"""Grouped convolution (csrc/gconv.cu) on the GPU: every production branch2b launch of ResNeXt-50 32x4d and 32x8d at
2 clips of 32 x 224^2 (fwd, dgrad, wgrad), and the ResNeXt-50 32x4d AVA FBO-NL training step next to the R50 step.

  python scripts/bench_gconv.py OUT_DIR [--iters 50] [--warmup 5] [--rounds 3] [--steps 10]

Per launch: CUDA-event time over `iters` back-to-back launches after `warmup`, algorithmic bytes (every operand and
result once) and FLOPs from the shapes, and the fraction of max(FLOP / 67 TFLOP/s, bytes / 3.35 TB/s) (H100 SXM data
sheet: FP32 non-tensor rate, HBM3 bandwidth) that the launch reaches, with the bound that decides it.  The two training
steps are timed alternately, `rounds` times each, `steps` CUDA-graph replays per timing.  Writes OUT_DIR/gconv.json
with the card name and power limit read in the same run.
"""
import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

FP32_FLOPS = 67e12
HBM_BYTES = 3.35e12


def card():
    import torch
    name = torch.cuda.get_device_name(0)
    try:
        out = subprocess.run(['nvidia-smi', '--query-gpu=power.limit', '--format=csv,noheader,nounits', '-i', '0'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        power = float(out.splitlines()[0])
    except Exception:
        power = None
    return name, power


def launch_table(iters, warmup):
    import torch
    import gconv_cases as GC
    rows = []
    for c in GC.CASES:
        if not c['name'].startswith('prod_'):
            continue
        t = GC.make_tensors(c, 'cuda')
        out = torch.zeros(t['out_shape'], dtype=torch.float32, device='cuda')
        bits = torch.zeros(out.numel() // 32, dtype=torch.int32, device='cuda') if c['epi'].get('bits') else None
        prm, keep = GC.prepare(c, t, out, bits)          # operands (dgrad: the grouped wt) built once, not timed
        for _ in range(warmup):
            GC.fire(prm)
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(iters):
            GC.fire(prm)
        e.record()
        e.synchronize()
        ms = s.elapsed_time(e) / iters
        g = GC.geom_of(c)
        G = c['groups']
        macs = g.N * g.To * g.Ho * g.Wo * g.Co * g.kT * g.kH * g.kW * (g.C // G)
        x_b, y_b, w_b = 4.0 * g.N * g.T * g.H * g.W * g.C, 4.0 * g.N * g.To * g.Ho * g.Wo * g.Co, 4.0 * macs / max(
            g.N * g.To * g.Ho * g.Wo, 1)
        if c['dir'] == 'fwd':
            nbytes = x_b + w_b + y_b + (y_b / 32 if bits is not None else 0)
        elif c['dir'] == 'dgrad':
            nbytes = y_b + w_b + x_b + x_b / 32        # dy, wt, dx, the ReLU sign bits of the mask
        else:
            nbytes = y_b + x_b + 2 * w_b               # dy, x, dw read and written by the accumulation
        flops = 2.0 * macs
        t_flop, t_byte = flops / FP32_FLOPS, nbytes / HBM_BYTES
        bound = 'fp32' if t_flop >= t_byte else 'hbm'
        frac = max(t_flop, t_byte) / (ms * 1e-3)
        rows.append(dict(name=c['name'], dir=c['dir'], ms=ms, gflop=flops / 1e9, mbytes=nbytes / 1e6,
                         tflops=flops / (ms * 1e-3) / 1e12, gbps=nbytes / (ms * 1e-3) / 1e9, bound=bound,
                         fraction_of_bound=frac))
        print('%-30s %8.3f ms  %6.1f GFLOP %8.1f MB  %5.1f TFLOP/s %6.0f GB/s  %s-bound  %4.0f%%' % (
            c['name'], ms, flops / 1e9, nbytes / 1e6, rows[-1]['tflops'], rows[-1]['gbps'], bound, 100 * frac))
        del keep, t, out, bits
        torch.cuda.empty_cache()
    return rows


def step_ms(resnext, steps, warmup):
    import numpy as np
    import torch
    import harness as H
    import resnext_oracle as RO
    from core.config import config as cfg
    from vlfb import workspace
    yaml = 'ava_r50_lfb_nl.yaml'
    ov = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2] + (['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4]
                                                   if resnext else [])
    H.setup_cfg(yaml, ov)
    cfg.RNG_SEED = 2
    workspace.ResetWorkspace()
    model, sfx = H.build('train', True)
    ocfg = H.oracle_cfg(yaml, ov)
    with RO.grouped() as OM:
        H.feed_params(OM.make_params(ocfg, seed=2))
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, seed=100)
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    for k, v in inputs.items():
        workspace.FeedBlob('gpu_0/%s%s' % (k, sfx), v.contiguous())
    name = model.net.Proto().name
    for _ in range(warmup):
        workspace.RunNet(name)
    torch.cuda.synchronize()
    s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    s.record()
    for _ in range(steps):
        workspace.RunNet(name)
    e.record()
    e.synchronize()
    loss = float(workspace.FetchBlob('gpu_0/loss'))
    assert np.isfinite(loss)
    workspace.ResetWorkspace()
    return s.elapsed_time(e) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('out_dir')
    ap.add_argument('--iters', type=int, default=50)
    ap.add_argument('--warmup', type=int, default=5)
    ap.add_argument('--rounds', type=int, default=3)
    ap.add_argument('--steps', type=int, default=10)
    args = ap.parse_args()
    import torch
    from vlfb import kernels as K
    K.set_gemm_backend('tcgen05')
    name, power = card()
    print('card: %s, power limit %s W' % (name, power))
    rows = launch_table(args.iters, args.warmup)
    steps = {'r50': [], 'resnext50_32x4d': []}
    for _ in range(args.rounds):
        for arm in ('r50', 'resnext50_32x4d'):
            ms = step_ms(arm != 'r50', args.steps, 3)
            steps[arm].append(ms)
            print('%-16s step %.2f ms = %.1f clips/s' % (arm, ms, 2000.0 / ms))
    summary = dict((arm, dict(ms=sorted(v), clips_per_s_median=2000.0 / sorted(v)[len(v) // 2]))
                   for arm, v in steps.items())
    os.makedirs(args.out_dir, exist_ok=True)
    with open(os.path.join(args.out_dir, 'gconv.json'), 'w') as f:
        json.dump(dict(card=name, power_limit_w=power, torch=torch.__version__, launches=rows, steps=summary,
                       clips_per_step=2), f, indent=1)
    print(json.dumps(dict(card=name, power_limit_w=power, steps=summary)))


if __name__ == '__main__':
    main()
