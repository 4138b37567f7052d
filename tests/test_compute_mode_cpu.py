"""B200.COMPUTE at CreateNet (CPU engine): 'tf32' lowers the net; any other value, the reserved 'fp32' included, raises
VlfbError instead of silently running the net in TF32."""
import pytest

import harness as H

TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4]


@pytest.fixture
def fake():
    import fake_kernels
    from vlfb import workspace
    fake_kernels.install()
    workspace.ResetWorkspace()
    yield fake_kernels
    workspace.ResetWorkspace()
    fake_kernels.uninstall()
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY)


def test_tf32_nets_are_created(fake):
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY + ['B200.COMPUTE', 'tf32'])
    model, _ = H.build('train', True)
    assert model.net.Proto().name


@pytest.mark.parametrize('value', ['fp32', 'bf16', 'TF32'])
def test_other_compute_values_are_refused(fake, value):
    from vlfb.libvlfb import VlfbError
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY + ['B200.COMPUTE', value])
    with pytest.raises(VlfbError, match='B200.COMPUTE'):
        H.build('train', True)
