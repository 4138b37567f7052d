#!/usr/bin/env python
"""Records the distinct launch signatures of the streaming kernels in one full-size training step.

The step is BASELINE config 2 (R50-I3D-NL + FBO-NL-2L, ava_r50_lfb_nl.yaml): 2 clips of 32x224x224, 2 RoIs per clip
(R = 4), a 300-row bank, run eagerly (no CUDA graph) so that every call goes through vlfb.kernels.  Each streaming
wrapper of vlfb.kernels (everything but the tensor-core GEMM wrappers, which tests/gemm_paths.py covers) is wrapped
for the step; a signature is the entry point with its shape, geometry and flag arguments
(tests/streaming_cases.signature).  The distinct signatures go to tests/golden/streaming_launches_config2.json,
which tests/test_streaming_cpu.py matches against the case table of tests/streaming_cases.py.

    python scripts/record_streaming_launches.py [--out FILE]      (needs an H100)
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'), ROOT, os.path.join(ROOT, 'tests')):
    if p not in sys.path:
        sys.path.insert(0, p)

YAML = 'ava_r50_lfb_nl.yaml'
CLIPS, ROIS_PER_CLIP = 2, 2


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', default=os.path.join(ROOT, 'tests', 'golden', 'streaming_launches_config2.json'))
    args = ap.parse_args(argv)
    import numpy as np
    import torch
    import harness as H
    import streaming_cases as SC
    from core.config import config as cfg
    from oracle import model as OM
    from vlfb import kernels as K
    from vlfb import workspace

    assert torch.cuda.is_available(), 'the step runs on the GPU'
    ov = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', CLIPS]
    H.setup_cfg(YAML, ov)
    cfg.RNG_SEED = 2
    cfg.B200.CUDA_GRAPH = False                 # eager: every launch goes through the wrappers
    workspace.ResetWorkspace()
    model, sfx = H.build('train', True)
    ocfg = H.oracle_cfg(YAML, ov)
    H.feed_params(OM.make_params(ocfg, seed=2))
    workspace.FeedBlob('gpu_0/lr', np.array(1e-4, dtype=np.float32))
    inputs = OM.make_inputs(ocfg, n_clips=CLIPS, rois_per_clip=ROIS_PER_CLIP, seed=100)

    def feed():                                 # every training step is fed a new clip (the layout launches of the feed)
        for k, v in inputs.items():
            workspace.FeedBlob('gpu_0/%s%s' % (k, sfx), v)
    name = model.net.Proto().name
    feed()
    workspace.RunNet(name)                      # first step: one-time preparation
    torch.cuda.synchronize()

    seen = {}
    saved = {}
    for fn in SC.STREAMING_WRAPPERS:
        orig = getattr(K, fn)
        saved[fn] = orig

        def wrapped(*a, _fn=fn, _orig=orig, **kw):
            sig = SC.signature(_fn, _orig, a, kw)
            key = json.dumps(sig, sort_keys=True)
            seen[key] = seen.get(key, 0) + 1
            return _orig(*a, **kw)
        setattr(K, fn, wrapped)
    try:
        feed()
        workspace.RunNet(name)
        torch.cuda.synchronize()
    finally:
        for fn, orig in saved.items():
            setattr(K, fn, orig)
    recs = [dict(json.loads(k), calls=n) for k, n in seen.items()]
    recs.sort(key=lambda r: (r['fn'], json.dumps(r['args'], sort_keys=True)))
    with open(args.out, 'w') as f:
        json.dump(dict(step='BASELINE config 2: %s, %d clips of 32x224x224, R = %d, L = 300, eager, second step with '
                            'its own input feed' % (YAML, CLIPS, CLIPS * ROIS_PER_CLIP),
                       device=torch.cuda.get_device_name(0), launches=recs), f, indent=1, sort_keys=True)
        f.write('\n')
    print('%d distinct streaming launch signatures (%d calls) -> %s' % (len(recs), sum(seen.values()), args.out))


if __name__ == '__main__':
    main()
