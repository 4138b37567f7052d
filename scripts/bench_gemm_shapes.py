"""Device-time table of the production GEMM shapes under the tiling / schedule variants of vlfb_gemm
(tile_n, stream_k).  Each entry = mean of `reps` back-to-back launches (CUDA events
around the batch; operands stay L2-resident as they are inside a training step)."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'))
from vlfb import kernels as K  # noqa: E402

REPS = int(os.environ.get('REPS', '20'))
VARIANTS = [('off', dict(pair=-1, stream_k=-1)), ('sk', dict(pair=-1, stream_k=1)), ('pair', dict(pair=1, stream_k=-1)),
            ('pair+sk', dict(pair=1, stream_k=1)), ('pair128+sk', dict(pair=1, stream_k=1, tile_n=128)),
            ('pair128', dict(pair=1, stream_k=-1, tile_n=128)), ('auto', dict())]
# name, Ci, Co, kernel, pads, dilation, (N, T, H, W)
CONVS = [
    ('res5_2b 3x3 512->512', 512, 512, (1, 3, 3), (0, 2, 2), (1, 2, 2), (2, 16, 14, 14)),
    ('res5_2a 3x1x1 2048->512', 2048, 512, (3, 1, 1), (1, 0, 0), (1, 1, 1), (2, 16, 14, 14)),
    ('res5_2a 1x1 2048->512', 2048, 512, (1, 1, 1), (0, 0, 0), (1, 1, 1), (2, 16, 14, 14)),
    ('res5_2c 1x1 512->2048', 512, 2048, (1, 1, 1), (0, 0, 0), (1, 1, 1), (2, 16, 14, 14)),
    ('res4_2b 3x3 256->256', 256, 256, (1, 3, 3), (0, 1, 1), (1, 1, 1), (2, 16, 14, 14)),
    ('res4_2a 3x1x1 1024->256', 1024, 256, (3, 1, 1), (1, 0, 0), (1, 1, 1), (2, 16, 14, 14)),
    ('res4_2c 1x1 256->1024', 256, 1024, (1, 1, 1), (0, 0, 0), (1, 1, 1), (2, 16, 14, 14)),
    ('res3_2b 3x3 128->128', 128, 128, (1, 3, 3), (0, 1, 1), (1, 1, 1), (2, 16, 28, 28)),
    ('res3_2a 3x1x1 512->128', 512, 128, (3, 1, 1), (1, 0, 0), (1, 1, 1), (2, 16, 28, 28)),
    ('res2_2b 3x3 64->64', 64, 64, (1, 3, 3), (0, 1, 1), (1, 1, 1), (2, 32, 56, 56)),
    ('res2_2c 1x1 64->256', 64, 256, (1, 1, 1), (0, 0, 0), (1, 1, 1), (2, 32, 56, 56)),
]


def timed(fn):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(REPS):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / REPS * 1e3      # us


def stem():
    """conv1 (5x7x7, stride 1x2x2, Cin 3 padded to 4) forward + weight gradient on a dense clip (16-byte cp.async gathers)
    and on the W-padded clip workspace feeds (TMA-staged overlapping-window operand)."""
    N, T, S = 2, 32, 224
    g = K.conv_geom((N, T, S, S, 4), 64, (5, 7, 7), (1, 2, 2), (2, 3, 3))
    w = torch.randn((64, 5, 7, 8, 4), device='cuda') * 0.05
    y = torch.empty(K.out_shape(g), device='cuda')
    dy = torch.randn(K.out_shape(g), device='cuda')
    dw = torch.zeros((64, 5, 7, 8, 4), device='cuda')
    s, b = torch.rand(64, device='cuda') + 0.5, torch.randn(64, device='cuda')
    dense = torch.randn((N, T, S, S, 4), device='cuda')
    pitch = 232
    buf = torch.zeros((N, T, S, pitch, 4), device='cuda')
    buf[:, :, :, 3:3 + S] = dense
    padded = buf[:, :, :, 3:3 + S]
    flop = 2.0 * y.numel() * 5 * 7 * 7 * 3 / 1e9
    for name, x in (('dense clip (cp.async)', dense), ('W-padded clip (TMA)', padded)):
        tf = timed(lambda: K.conv_fwd(x, w, y, g, scale=s, bias=b, relu=True, tf32_out=True))
        tw = timed(lambda: K.conv_wgrad(dy, x, dw, g, row_scale=s))
        print('conv1 %-24s fwd %8.1fus (%6.1f TF/s)   wgrad %8.1fus (%6.1f TF/s)' % (name, tf, flop / tf * 1e3, tw, flop / tw * 1e3),
              flush=True)


def strided():
    """The networks' stride-2 layers: data gradient (parity classes on the tensor-core engine; VLFB_NO_PAR=1 = the
    cp.async gather over all taps), plain and as the finishing contribution (+ residual, ReLU mask, TF32 rounding)."""
    for name, ci, co, ker, pd, shp in [('res3_0_2b 3x3/2 128->128', 128, 128, (1, 3, 3), (0, 1, 1), (2, 16, 56, 56)),
                                       ('res4_0_2b 3x3/2 256->256', 256, 256, (1, 3, 3), (0, 1, 1), (2, 16, 28, 28)),
                                       ('res3_0_b1 1x1/2 256->512', 256, 512, (1, 1, 1), (0, 0, 0), (2, 16, 56, 56)),
                                       ('res4_0_b1 1x1/2 512->1024', 512, 1024, (1, 1, 1), (0, 0, 0), (2, 16, 28, 28))]:
        g = K.conv_geom(shp + (ci,), co, ker, (1, 2, 2), pd, (1, 1, 1))
        taps = ker[0] * ker[1] * ker[2]
        wt = torch.randn((ci, taps, co), device='cuda') * 0.05
        dy = torch.randn(K.out_shape(g), device='cuda')
        dx = torch.empty(shp + (ci,), device='cuda')
        res, mask = torch.randn_like(dx), torch.randn_like(dx)
        flop = 2.0 * dy.numel() * taps * ci / 1e9
        t0 = timed(lambda: K.conv_dgrad(dy, wt, dx, g))
        t1 = timed(lambda: K.conv_dgrad(dy, wt, dx, g, residual=res, relu_mask=mask, tf32_out=True))
        print('%-28s dgrad %8.1fus (%6.1f TF/s)   finishing dgrad %8.1fus' % (name, t0, flop / t0 * 1e3, t1), flush=True)


def epilogue_bound():
    """Large-M, short-K layers (res2): the epilogue streams are the bound.  GB/s = algorithmic bytes / time."""
    shp = (2, 32, 56, 56)
    M = shp[0] * shp[1] * shp[2] * shp[3]
    for name, ci, co, ker, pd in [('res2_2c 1x1 64->256', 64, 256, (1, 1, 1), (0, 0, 0)),
                                  ('res2_2a 3x1x1 256->64', 256, 64, (3, 1, 1), (1, 0, 0))]:
        g = K.conv_geom(shp + (ci,), co, ker, (1, 1, 1), pd, (1, 1, 1))
        taps = ker[0]
        x = torch.randn(shp + (ci,), device='cuda')
        w = torch.randn((co,) + ker + (ci,), device='cuda') * 0.05
        wt = torch.randn((ci, taps, co), device='cuda') * 0.05
        s, b = torch.rand(co, device='cuda') + 0.5, torch.randn(co, device='cuda')
        y = torch.empty(K.out_shape(g), device='cuda')
        dy = torch.randn(K.out_shape(g), device='cuda')
        dx = torch.empty(shp + (ci,), device='cuda')
        resy = torch.randn_like(y)
        res, mask = torch.randn_like(dx), torch.randn_like(dx)
        mbits = torch.empty((dx.numel() // 32,), dtype=torch.int32, device='cuda')
        K.relu_bits(mask, mbits)
        ybits = torch.empty((y.numel() // 32,), dtype=torch.int32, device='cuda')
        cases = [('fwd', lambda: K.conv_fwd(x, w, y, g, scale=s, bias=b, relu=True, tf32_out=True), M * (ci + co) * 4),
                 ('fwd+res', lambda: K.conv_fwd(x, w, y, g, scale=s, bias=b, residual=resy, relu=True, tf32_out=True), M * (ci + 2 * co) * 4),
                 ('dgrad', lambda: K.conv_dgrad(dy, wt, dx, g), M * (ci + co) * 4),
                 ('dgrad+res', lambda: K.conv_dgrad(dy, wt, dx, g, residual=res, tf32_out=True), M * (2 * ci + co) * 4),
                 ('dgrad+res+mask', lambda: K.conv_dgrad(dy, wt, dx, g, residual=res, relu_mask=mask, tf32_out=True), M * (3 * ci + co) * 4),
                 ('dgrad+res+bits', lambda: K.conv_dgrad(dy, wt, dx, g, residual=res, relu_mask_bits=mbits, tf32_out=True),
                  M * (2 * ci + co) * 4 + M * ci / 8),
                 ('fwd+res+bits out', lambda: K.conv_fwd(x, w, y, g, scale=s, bias=b, residual=resy, relu=True, tf32_out=True, relu_bits=ybits),
                  M * (ci + 2 * co) * 4 + M * co / 8)]
        for cname, fn, nbytes in cases:
            t = timed(fn)
            print('%-24s %-16s %8.1fus  %7.0f GB/s' % (name, cname, t, nbytes / t / 1e3), flush=True)


def main():
    only = sys.argv[1:] or None
    if not only or 'conv1' in only:
        stem()
    if only and 'strided' in only:
        strided()
    if only and 'epi' in only:
        epilogue_bound()
    if only and all(o in ('conv1', 'strided', 'epi') for o in only):
        return
    print('%-28s %-6s' % ('layer', 'op') + ''.join('%12s' % n for n, _ in VARIANTS) + '   GFLOP   best TF/s')
    for name, ci, co, ker, pd, dil, shp in CONVS:
        if only and not any(o in name for o in only):
            continue
        g = K.conv_geom(shp + (ci,), co, ker, (1, 1, 1), pd, dil)
        x = torch.randn(shp + (ci,), device='cuda')
        w = torch.randn((co,) + ker + (ci,), device='cuda') * 0.05
        taps = ker[0] * ker[1] * ker[2]
        wt = torch.randn((ci, taps, co), device='cuda') * 0.05
        s, b = torch.rand(co, device='cuda') + 0.5, torch.randn(co, device='cuda')
        y = torch.empty(K.out_shape(g), device='cuda')
        dy = torch.randn(K.out_shape(g), device='cuda')
        dx = torch.empty(shp + (ci,), device='cuda')
        dw = torch.zeros((co,) + ker + (ci,), device='cuda')
        flop = 2.0 * y.numel() * taps * ci / 1e9
        ops = [('fwd', lambda: K.conv_fwd(x, w, y, g, scale=s, bias=b, relu=True, tf32_out=True)),
               ('dgrad', lambda: K.conv_dgrad(dy, wt, dx, g)),
               ('wgrad', lambda: K.conv_wgrad(dy, x, dw, g, row_scale=s))]
        for opname, fn in ops:
            row = []
            for _, opts in VARIANTS:
                K.GEMM_OPTS.update(dict(tile_n=0, pair=0, stream_k=0))
                K.GEMM_OPTS.update(opts)
                row.append(timed(fn))
            K.GEMM_OPTS.update(dict(tile_n=0, pair=0, stream_k=0))
            print('%-28s %-6s' % (name, opname) + ''.join('%10.1fus' % t for t in row) +
                  '  %6.1f  %8.1f' % (flop, flop / min(row) * 1e3), flush=True)


if __name__ == '__main__':
    main()
