"""Times representative hot-path GEMM launches under kernel tuning overrides (VLFB_BN / VLFB_STAGES /
VLFB_LAG / VLFB_TMA environment variables read by gemm_tc.cu at launch).  Prints one line per (shape, config)."""
import itertools
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'))
from vlfb import kernels as K  # noqa: E402


def make(N, T, H, W, Ci, Co, ker, st, pd, dil):
    g = K.conv_geom((N, T, H, W, Ci), Co, ker, st, pd, dil)
    x = torch.randn((N, T, H, W, Ci), device='cuda')
    w = torch.randn((Co,) + tuple(ker) + (Ci,), device='cuda') * 0.05
    y = torch.randn(K.out_shape(g), device='cuda')
    taps = ker[0] * ker[1] * ker[2]
    wt = torch.randn((Ci, taps, Co), device='cuda') * 0.05
    return g, x, w, y, wt


SHAPES = {
    'res5_2b 3x3d2 512->512': (2, 16, 14, 14, 512, 512, (1, 3, 3), (1, 1, 1), (0, 2, 2), (1, 2, 2)),
    'res4_2b 3x3 256->256': (2, 16, 14, 14, 256, 256, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1)),
    'res4_2c 1x1 256->1024': (2, 16, 14, 14, 256, 1024, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1)),
    'res3_2a 3x1x1 512->128': (2, 16, 28, 28, 512, 128, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1)),
    'res2_2c 1x1 64->256': (2, 32, 56, 56, 64, 256, (1, 1, 1), (1, 1, 1), (0, 0, 0), (1, 1, 1)),
    'res2_2b 3x3 64->64': (2, 32, 56, 56, 64, 64, (1, 3, 3), (1, 1, 1), (0, 1, 1), (1, 1, 1)),
    'res2_2a 3x1x1 256->64': (2, 32, 56, 56, 256, 64, (3, 1, 1), (1, 1, 1), (1, 0, 0), (1, 1, 1)),
}


def timeit(fn, reps=5):
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def main():
    configs = [dict(), dict(VLFB_LAG='1'), dict(VLFB_LAG='3'), dict(VLFB_TMA='0')]
    for name, shp in SHAPES.items():
        g, x, w, y, wt = make(*shp)
        dw = torch.zeros_like(w)
        dx = torch.empty_like(x)
        flops = 2.0 * g.N * g.To * g.Ho * g.Wo * g.Co * g.C * g.kT * g.kH * g.kW
        for cfg in configs:
            for k in ('VLFB_BN', 'VLFB_STAGES', 'VLFB_LAG', 'VLFB_TMA'):
                os.environ.pop(k, None)
            os.environ.update(cfg)
            tf = timeit(lambda: K.conv_fwd(x, w, y, g, relu=True, tf32_out=True))
            td = timeit(lambda: K.conv_dgrad(y, wt, dx, g))
            tw = timeit(lambda: K.conv_wgrad(y, x, dw, g))
            print('%-26s %-44s fwd %7.3f ms %6.1f TF | dgrad %7.3f ms %6.1f TF | wgrad %7.3f ms %6.1f TF' % (
                name, ' '.join('%s=%s' % (k[5:], v) for k, v in cfg.items()) or 'default', tf, flops / tf / 1e9,
                td, flops / td / 1e9, tw, flops / tw / 1e9), flush=True)


if __name__ == '__main__':
    main()
