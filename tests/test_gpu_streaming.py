"""The streaming kernels (csrc/ops.cu, csrc/fbo.cu) against fp64, case by case (tests/streaming_cases.py): elementwise
bounds or bit-exactness, untouched guard bands, determinism where the ABI promises it, and every production launch of
a config-2 training step at its recorded shape."""
import collections

import pytest
import torch

import streaming_cases as SC

pytestmark = pytest.mark.gpu
_WORST = collections.defaultdict(float)


@pytest.fixture(scope='module')
def K():
    from vlfb import kernels
    yield kernels
    for fn in sorted(_WORST):             # the worst |got - ref| / bound of each family (0: bit-exact) over the cases run
        print('[streaming] %-22s worst bound ratio %.3g' % (fn, _WORST[fn]))


@pytest.mark.parametrize('name', [c['name'] for c in SC.CASES])
def test_streaming_case(K, name):
    c = SC.case_by_name(name)
    if c['fn'] == 'fbo_bank_scan':        # the table's split counts are the library's
        from vlfb import libvlfb as L
        R, Lr, D = c['args']['bank']['shape']
        bf16 = c['args']['bank']['dtype'] == 'bfloat16'
        assert L.load().vlfb_fbo_bank_scan_splits_dt(R, Lr, D, L.DT_BF16 if bf16 else L.DT_F32) == \
            SC.scan_splits(R, Lr, D, bf16)
    rec = SC.check_case(K, c, torch.device('cuda'))
    _WORST[rec['fn']] = max(_WORST[rec['fn']], rec['worst_ratio'])
    print('[streaming] %s worst bound ratio %.3g' % (name, rec['worst_ratio']))
    assert rec['ok'], '%s: %s' % (name, '; '.join(rec['errors']))
