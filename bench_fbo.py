#!/usr/bin/env python
"""bench_fbo.py -- BASELINE.json configs[4]: Feature-Bank-Operator (FBO-NL) microbenchmark on one H100.

Sweeps the bank length L and the RoI count R over the FBO-NL head alone (lfb_helper.add_fbo_nl_head: query
reduction 2048->512, bank projection 'lfb_1x1', NUM_LAYERS single-query non-local layers), built through the same
builder API / workspace / C ABI as the full model, in three modes:

  infer_fold   test-mode graph, every layer = ONE pass over the raw bank (executor.FboFoldStep + fbo_bank_scan): HBM-bound
  infer_fold_bf16  the same with the bank stored as bf16 (B200.LFB_DTYPE; fp32 scores / softmax / sums): half the bytes
  infer        test-mode graph as written (B200.FBO_FOLD False): bank projections on the tensor-core GEMM
  train        train-mode graph (dropout on) forward + backward + SGD, as written

One JSON line per (mode, R, L, layers) on stdout:
  ms = device time of the captured step (CUDA-graph replay bracketed by events; runnet_ms = the same through
  workspace.RunNet, which adds ~0.2 ms of python per call and is what bounds tiny cases), GB/s = SURVEY 8(d) compulsory bytes / time, against MEASURED_PEAKS.json hbm_gbs; TFLOP/s = as-written FLOPs / time
  (for infer_fold this is "effective" throughput: the folded path does not execute those FLOPs);
  scan = the fbo_bank_scan launches alone (CUDA events around each, eager pass): achieved GB/s of the dominant kernel.
Inputs are resident in HBM; L2 is flushed (256 MB write) before every timed iteration, so a bank that would fit the
50 MB L2 is still read from HBM once per iteration.
"""
import argparse
import json
import os
import sys
import types

ROOT = os.path.dirname(os.path.abspath(__file__))
for p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

YAML = {2: 'ava_r50_lfb_nl.yaml', 3: 'ava_r50_lfb_nl_3l.yaml'}
STATE = {'L': 300}


def fbo_bytes(R, L, layers, s=4, bank_s=None):
    """SURVEY.md 8(d): compulsory bytes of the FBO-NL block (bank + box_pooled + out + weights/biases); `bank_s` =
    bytes per bank element when the bank's storage type differs from the rest (bf16 bank, fp32 weights)."""
    bank_s = s if bank_s is None else bank_s
    return bank_s * R * L * 2048 + s * (R * 2048 + R * 512) + s * (2 * 2048 * 512 + layers * 4 * 512 ** 2 + (2 + 4 * layers) * 512)


def fbo_flops(R, L, layers):
    """SURVEY.md 8(d): forward FLOPs of the block as written."""
    return 2.0 * R * (2048 * 512 + L * 2048 * 512 + layers * (2 * 512 ** 2 + 2 * L * 512 ** 2 + 2 * L * 512))


def _creator():
    """FBO-NL head + classifier as a model creator (same call sequence as resnet_video.create_model :300-349 after
    the backbone: head_helper.add_roi_head's FBO branch -> FC 'pred' -> loss)."""
    from core.config import config as cfg
    from models import lfb_helper

    def create_model(model, data, labels, split, lfb_infer_only, suffix):
        test_mode = split in ('test', 'val')
        blob, dim = lfb_helper.add_fbo_nl_head(model, data, 2048, STATE['L'], test_mode, suffix)
        logits = model.FC(blob, 'pred', dim, cfg.MODEL.NUM_CLASSES,
                          weight_init=('GaussianFill', {'std': cfg.MODEL.FC_INIT_STD}),
                          bias_init=('ConstantFill', {'value': 0.}))
        if split == 'train':
            prob = model.Sigmoid(logits, 'prob')
            loss = model.SigmoidCrossEntropyLoss([logits, labels], ['loss'], scale=1. / cfg.NUM_GPUS)
            return model, prob, loss
        return model, model.Sigmoid(logits, 'prob', engine='CUDNN'), None
    return types.SimpleNamespace(create_model=create_model)


def build_case(mode, R, L, layers):
    """Build + feed the FBO-only net; returns (model, net name)."""
    import numpy as np
    import torch
    import harness as H
    from core.config import config as cfg
    from models import model_builder_video as MB
    from vlfb import workspace

    train = mode == 'train'
    H.setup_cfg(YAML[layers], ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TEST.BATCH_SIZE', 2])
    cfg.MODEL.MODEL_NAME = 'fbo_nl_only'
    cfg.B200.FBO_FOLD = mode.startswith('infer_fold')
    cfg.B200.LFB_DTYPE = 'bf16' if mode.endswith('_bf16') else 'f32'
    cfg.RNG_SEED = 2
    MB.model_creator_map['fbo_nl_only'] = _creator()
    STATE['L'] = L
    workspace.ResetWorkspace()
    model, sfx = H.build('train' if train else 'val', train)
    g = torch.Generator().manual_seed(3)
    # zero-initialised `out` convs (the reference's init) would make the layers no-ops numerically but not in time;
    # give them Gaussian weights so that the timed data flow is the trained model's
    for l in range(layers):
        shape = workspace.current().params.logical_shape('lfb_nl%d_out_w' % l)
        workspace.FeedBlob('gpu_0/lfb_nl%d_out_w' % l, (torch.randn(shape, generator=g) * 0.02).numpy())
    uniq = min(R, 16)                       # distinct RoI banks; repeated along R (timing does not depend on values)
    bank = torch.randn((uniq, L, 2048), generator=g) * 0.5
    bank[:, L - (L + 3) // 4:] = 0.0
    bank = bank.repeat((R + uniq - 1) // uniq, 1, 1)[:R].contiguous()
    workspace.FeedBlob('gpu_0/data' + sfx, torch.relu(torch.randn((R, 2048, 1, 1, 1), generator=g)).numpy())
    workspace.FeedBlob('gpu_0/lfb' + sfx, bank.numpy())
    workspace.FeedBlob('gpu_0/labels' + sfx, (torch.rand((R, cfg.MODEL.NUM_CLASSES), generator=g) < 0.05).to(torch.int32).numpy())
    del bank
    if train:
        workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    return model, model.net.Proto().name


def run_case(mode, R, L, layers, steps, warmup, peaks):
    import numpy as np
    import torch
    from vlfb import kernels as K
    from vlfb import workspace

    train = mode == 'train'
    model, name = build_case(mode, R, L, layers)
    flush = torch.empty(64 * 1024 * 1024, dtype=torch.float32, device='cuda')
    for _ in range(max(warmup, 3)):
        workspace.RunNet(name)
    torch.cuda.synchronize()
    net = workspace.current().nets[name]
    assert len(net._graphs) == 1, 'the step should have been captured after the warm-up runs'
    g1, g2, n1, n2 = list(net._graphs.values())[0][:4]

    def timed(fn):
        evs = []
        for _ in range(steps):
            flush.zero_()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            fn()
            e1.record()
            evs.append((e0, e1))
        torch.cuda.synchronize()
        return sorted(a.elapsed_time(b) for a, b in evs)

    def replay():                 # the captured step itself: what the device executes, without RunNet's host work
        g1.replay()
        if g2 is not None:
            g2.replay()

    K.LAUNCHES = 0
    api_times = timed(lambda: workspace.RunNet(name))
    launches = K.LAUNCHES // max(steps, 1)
    times = timed(replay)
    ms = times[len(times) // 2]
    api_ms = api_times[len(api_times) // 2]
    out = float(np.abs(workspace.FetchBlob('gpu_0/prob')).sum())
    assert np.isfinite(out)
    # the dominant kernel alone (eager pass with per-launch events)
    scan = None
    workspace.current().force_eager = True
    flush.zero_()
    K.start_profile()
    workspace.RunNet(name)
    recs = K.stop_profile()
    workspace.current().force_eager = False
    srecs = [r for r in recs if r[0].startswith('fbo_bank_scan')]
    if srecs:
        t = sum(r[1] for r in srecs)
        scan = {'launches': len(srecs), 'ms': round(t, 4), 'alg_bytes_per_launch': srecs[0][3],
                'gbs': round(sum(r[3] for r in srecs) / 1e6 / t, 1), 'frac': round(sum(r[3] for r in srecs) / 1e6 / t / peaks['hbm_gbs'], 3)}
    gemm_ms = sum(r[1] for r in recs if not r[0].startswith('fbo_bank_scan'))
    bf16 = mode.endswith('_bf16')
    nbytes = fbo_bytes(R, L, layers, bank_s=2 if bf16 else 4)
    flops = fbo_flops(R, L, layers) * (3.0 if train else 1.0)
    workspace.ResetWorkspace()
    torch.cuda.empty_cache()
    return {'bench': 'fbo_nl', 'mode': mode, 'R': R, 'L': L, 'layers': layers, 'ms': round(ms, 4), 'ms_min': round(times[0], 4),
            'runnet_ms': round(api_ms, 4),
            'launches': launches, 'alg_bytes': nbytes, 'gbs': round(nbytes / 1e6 / ms, 1),
            'hbm_frac': round(nbytes / 1e6 / ms / peaks['hbm_gbs'], 4), 'as_written_gflop': round(flops / 1e9, 2),
            'tflops_as_written': round(flops / 1e9 / ms, 1), 'scan': scan, 'gemm_ms_eager': round(gemm_ms, 4),
            'rois_per_s': round(R / ms * 1e3, 0),
            'dtype': 'tf32' if not mode.startswith('infer_fold') else ('bf16 bank, ' if bf16 else '') + 'f32 scan + tf32 R-row matmuls',
            'l2': 'flushed before every iteration', 'cuda_graph': True}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--R', default='4,16,64,256')
    ap.add_argument('--L', default='60,300,1200,3600')
    ap.add_argument('--layers', default='2,3')
    ap.add_argument('--modes', default='infer_fold,infer_fold_bf16,infer,train')
    ap.add_argument('--steps', type=int, default=20)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--max-rows', type=int, default=256 * 3600, help='skip cases with R*L above this')
    ap.add_argument('--out', default='')
    args = ap.parse_args()
    import torch
    assert torch.cuda.is_available(), 'bench_fbo.py needs a GPU (there is no CPU path)'
    try:
        with open(os.path.join(ROOT, 'MEASURED_PEAKS.json')) as f:
            peaks = json.load(f)
    except Exception:
        peaks = {'hbm_gbs': 3350.0, 'bf16_tflops_sustained': 989.0}     # H100 SXM data sheet (dense, 700 W card)
    rows = []
    for layers in [int(v) for v in args.layers.split(',')]:
        for mode in args.modes.split(','):
            for R in [int(v) for v in args.R.split(',')]:
                for L in [int(v) for v in args.L.split(',')]:
                    if R * L > args.max_rows or (mode == 'train' and R * L > args.max_rows // 4):
                        continue
                    r = run_case(mode, R, L, layers, args.steps, args.warmup, peaks)
                    rows.append(r)
                    print(json.dumps(r), flush=True)
    if args.out:
        with open(args.out, 'w') as f:
            f.write('# FBO-NL microbench (bench_fbo.py), HBM peak %.0f GB/s (MEASURED_PEAKS.json)\n' % peaks['hbm_gbs'])
            f.write('%-11s %4s %5s %2s %9s %9s %8s %8s %9s %7s  %s\n' % ('mode', 'R', 'L', 'l', 'ms', 'runnet_ms', 'GB/s', 'hbm_frac',
                                                                      'TF/s(aw)', 'launch', 'scan kernel GB/s (frac)'))
            for r in rows:
                sc = '%.0f (%.2f)' % (r['scan']['gbs'], r['scan']['frac']) if r['scan'] else '-'
                f.write('%-11s %4d %5d %2d %9.4f %9.4f %8.0f %8.3f %9.1f %7d  %s\n' % (
                    r['mode'], r['R'], r['L'], r['layers'], r['ms'], r['runnet_ms'], r['gbs'], r['hbm_frac'],
                    r['tflops_as_written'], r['launches'], sc))


if __name__ == '__main__':
    main()
