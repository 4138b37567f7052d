"""Every kernel launch of real steps, audited on the GPU (tests/launch_audit.py): the tiny nets run eagerly
(B200.CUDA_GRAPH off, the optimizer update included, train nets twice) and every call of a vlfb.kernels wrapper is
checked against fp64 from its own tensors, with the TF32-exactness check of the GEMM operands on the tensor-core
engine.  Each net runs in its own process with VLFB_DEBUG set, so every GEMM record carries its launch's path.

The full-size config-2 step (the benchmarked one) runs once unaudited, then once audited, every call, within a
ten-minute budget."""
import time

import pytest

import launch_audit as LA
from util import run_worker

pytestmark = pytest.mark.gpu

GPU_NETS = ['ava_train', 'ava_train_simt', 'ava_train_dropout', 'charades_train', 'charades_softmax_train',
            'ava_val_fold_f32', 'ava_val_fold_bf16', 'ava_lfb_infer_only', 'ava_train_det', 'ava_train_capacity',
            'resnext_bn_train', 'resnext_bn_train_det', 'config2_train']
# wall-time budget of one net's audit, process start included: a minute per tiny net, ten for the full-size step
BUDGET_S = dict(config2_train=600.0)


@pytest.mark.parametrize('net', GPU_NETS)
def test_every_launch_of_a_tiny_net_matches_fp64(net):
    t0 = time.time()
    p, recs = run_worker('launch_audit.py', ['--net', net], timeout=1200)
    wall = time.time() - t0
    print('\n[%s] wall %.1f s\n%s' % (net, wall, p.stdout[-4000:]))
    assert p.returncode == 0, p.stderr[-4000:]
    *recs, tail = recs
    assert not tail['missing'], 'wrappers the net never reached: %s' % tail['missing']
    bad = [r for r in recs if not r['ok']]
    assert not bad, '\n'.join(e for r in bad[:20] for e in r['errors'])
    assert {r['run'] for r in recs} - {0} == set(range(1, LA.NETS[net][3] + 1))      # run 0: feeding the blobs
    if LA.NETS[net][5].get('backend', 'tcgen05') == 'tcgen05':
        gemm = [r for r in recs if r['wrapper'] in LA.GEMM_WRAPPERS]
        assert gemm and all(r.get('paths') for r in gemm if r['wrapper'].startswith('conv')), \
            'tensor-core GEMM calls without a path record'
    budget = BUDGET_S.get(net, 60.0)
    assert wall < budget, 'the audit of %s took %.0f s (budget %.0f s)' % (net, wall, budget)

