"""CPU checks of grouped convolution (ResNeXt `RESNETS.NUM_GROUPS`): the C ABI's rules for vlfb_gemm_params_t.groups,
the case table of tests/gconv_cases.py and its comparison (which must reject planted errors), a TINY ResNeXt net
recorded through the builder API and lowered by the executor against the fp64 oracle on the torch-CPU kernels, and
the checkpoint round trip of grouped weights."""
import ctypes
import os
import pickle

import numpy as np
import pytest
import torch

import gconv_cases as GC
import harness as H
import resnext_oracle as RO

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RESNEXT = ['RESNETS.NUM_GROUPS', 32, 'RESNETS.WIDTH_PER_GROUP', 4]
TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8,
        'TEST.BATCH_SIZE', 2, 'TEST.CROP_SIZE', 64, 'TEST.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]


# ------------------------------------------------------------------------------------------------ C ABI
def test_groups_field_offset_matches_header(tmp_path):
    import subprocess
    from vlfb import libvlfb as L
    src = tmp_path / 'g.c'
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "vlfb.h"\nint main(void) {\n'
                   '  printf("%zu %zu\\n", offsetof(vlfb_gemm_params_t, groups), sizeof(vlfb_gemm_params_t));\n'
                   '  return 0;\n}\n')
    exe = tmp_path / 'g'
    subprocess.check_call(['gcc', '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
    off, size = [int(v) for v in subprocess.check_output([str(exe)]).decode().split()]
    assert off == L.GemmParams.groups.offset and size == ctypes.sizeof(L.GemmParams)


@pytest.mark.parametrize('rule', sorted(GC.ABI_RULES))
def test_abi_rejects(rule):
    """Each invalid combination fails validation (before any device access) with its message."""
    from vlfb import libvlfb as L
    lib = L.load()
    p, code, needle = GC.ABI_RULES[rule]()
    assert lib.vlfb_gemm(ctypes.byref(p), None) == code, (rule, lib.vlfb_last_error())
    assert needle.encode() in lib.vlfb_last_error(), (rule, lib.vlfb_last_error())


def test_plan_query_refuses_groups():
    from vlfb import libvlfb as L
    lib = L.load()
    p = GC._base()                      # a valid grouped fwd: vlfb_gemm would accept it
    plan = L.GemmPlan()
    assert lib.vlfb_gemm_plan(ctypes.byref(p), 132, ctypes.byref(plan)) == -2
    assert b'grouped' in lib.vlfb_last_error()


# ------------------------------------------------------------------------------------------------ case table
def test_case_table_is_well_formed():
    GC.check_table()


@pytest.mark.parametrize('plant', sorted(GC.PLANTS))
def test_comparison_rejects_planted_error(plant):
    """The elementwise bound must catch each planted kernel bug on a case that exercises it."""
    case, bad_fn = GC.PLANTS[plant]
    ok, _ = GC.run_case_cpu(case)
    assert ok, plant
    ok, why = GC.run_case_cpu(case, plant=bad_fn)
    assert not ok, plant


# ------------------------------------------------------------------------------------------------ engine
@pytest.fixture
def fake():
    from vlfb import workspace
    RO.install()
    workspace.ResetWorkspace()
    yield RO
    workspace.ResetWorkspace()
    RO.uninstall()


def test_conv_nd_rejects_unsupported_widths():
    from vlfb.cnn import CNNModelHelper
    m = CNNModelHelper()
    with pytest.raises(ValueError, match='multiples of 4'):
        m.ConvNd('x', 'c', 64, 64, [1, 3, 3], group=32)         # 2 channels per group
    with pytest.raises(ValueError, match='multiples of 4'):
        m.ConvNd('x', 'c', 256, 256, [1, 3, 3], group=2)        # 128 channels per group
    with pytest.raises(ValueError, match='1x1x1'):
        m.ConvNd('x', 'c', 128, 128, [1, 1, 1], group=32)
    m.ConvNd('x', 'ok', 128, 128, [1, 3, 3], group=32)
    shapes = dict((op.outputs[0], list(op.args['shape'])) for op in m.param_init_net.Proto().op if 'shape' in op.args)
    assert shapes['ok_w'] == [128, 4, 1, 3, 3]


def test_tiny_resnext_records_caffe2_shapes_and_lowers_per_group(fake):
    from vlfb import executor as X
    from vlfb import workspace
    ov = TINY + RESNEXT
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    with RO.grouped() as OM:
        spec = OM.param_spec(ocfg)
    assert spec['res2_0_branch2b_w'][0] == (128, 4, 1, 3, 3)
    assert spec['res5_0_branch2b_w'][0] == (1024, 32, 1, 3, 3)
    model, _ = H.build('train', True)
    shapes = dict((op.outputs[0], list(op.args['shape'])) for op in model.param_init_net.Proto().op
                  if 'shape' in op.args)
    for name, (shape, _) in spec.items():
        if name in shapes:
            assert tuple(shapes[name]) == tuple(shape), name
    net = workspace.current().nets[model.net.Proto().name]
    grouped = [st for st in net.steps if isinstance(st, X.ConvStep) and st.groups > 1]
    assert len(grouped) == 16 and all(st.affine is not None and st.relu for st in grouped)
    assert all(st.op.inputs[1].endswith('branch2b_w') for st in grouped)


def test_tiny_resnext_train_matches_oracle(fake):
    """Forward blobs, loss and every parameter gradient in fp64 (both gradient-sum schedules), then one SGD step."""
    import test_engine_cpu as E
    from vlfb import executor as X
    from vlfb import workspace
    with RO.grouped():
        model, params, p64, worst = E._run('ava_r50_lfb_nl.yaml', TINY + RESNEXT, fake,
                                           ['res2_2_branch2c_bn', 'res3_3_branch2c_bn', 'res5_2_branch2c_bn',
                                            'box_pooled', 'pred'], reps=2)
    net = workspace.current().nets[model.net.Proto().name]
    jobs = net._wt_jobs
    grouped = [st for st in net.steps if isinstance(st, X.ConvStep) and st.groups > 1 and id(st) in net.wt_buffers]
    # one weight-transpose job per group of every grouped conv whose input needs a gradient
    plain = [st for st in net.steps if isinstance(st, X.ConvStep) and st.groups == 1 and id(st) in net.wt_buffers]
    assert len(grouped) > 0 and len(jobs) == len(plain) + 32 * len(grouped)


def test_tiny_resnext_val_split_matches_oracle(fake):
    from vlfb import workspace
    ov = TINY + RESNEXT
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    with RO.grouped() as OM:
        params = OM.make_params(ocfg, seed=2, split='val')
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=3, crop=64, frames=8)
        blobs, _, _ = OM.forward(ocfg, params, inputs, 'val')
    model, sfx = H.build('val', False)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    workspace.RunNet(model.net.Proto().name)
    for b in ('res5_2_branch2c_bn', 'box_pooled', 'pred'):
        assert H.rel(workspace.FetchBlob('gpu_0/' + b), blobs[b].numpy()) < 1e-5, b


# ------------------------------------------------------------------------------------------------ checkpoints
def test_grouped_weights_checkpoint_round_trip(fake, tmp_path):
    """Save after one SGD step, reload into a fresh net: grouped weights and their momentum keep the Caffe2 shape."""
    from utils import checkpoints as CK
    from vlfb import workspace
    ov = TINY + RESNEXT
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    ocfg = H.oracle_cfg('ava_r50_lfb_nl.yaml', ov)
    with RO.grouped() as OM:
        params = OM.make_params(ocfg, seed=2)
        inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=2, crop=64, frames=8)
    model, sfx = H.build('train', True)
    H.feed_params(params)
    H.feed_inputs(inputs, sfx)
    model.UpdateWorkspaceLr(10)
    workspace.RunNet(model.net.Proto().name)
    w = workspace.FetchBlob('gpu_0/res3_0_branch2b_w').copy()
    mo = workspace.FetchBlob('gpu_0/res3_0_branch2b_w_momentum').copy()
    assert w.shape == (256, 8, 1, 3, 3) and np.abs(mo).max() > 0
    path = str(tmp_path / 'c2_model_iter10.pkl')
    CK.save_model_params(model, path, 9)
    with open(path, 'rb') as f:
        blobs = pickle.load(f, encoding='latin1')['blobs']
    np.testing.assert_allclose(blobs['res3_0_branch2b_w'], w, rtol=1e-6, atol=0)       # stored as fp32
    workspace.ResetWorkspace()
    H.setup_cfg('ava_r50_lfb_nl.yaml', ov)
    model2, _ = H.build('train', True)
    it, _ = CK.initialize_params_from_file(model2, path)
    assert it == 10
    # the checkpoint loader feeds fp32, as the reference's
    np.testing.assert_allclose(workspace.FetchBlob('gpu_0/res3_0_branch2b_w'), w, rtol=1e-6, atol=0)
    np.testing.assert_allclose(workspace.FetchBlob('gpu_0/res3_0_branch2b_w_momentum'), mo, rtol=1e-6, atol=0)


def test_2d_resnext_weights_inflate(fake, tmp_path):
    """An ImageNet ResNeXt pickle holds 2-D branch2b weights [Co, Cig, kH, kW]: they load as [Co, Cig, 1, kH, kW]."""
    from utils import checkpoints as CK
    from vlfb import workspace
    H.setup_cfg('ava_r50_lfb_nl.yaml', TINY + RESNEXT)
    model, _ = H.build('train', True)
    w2d = np.random.RandomState(0).randn(128, 4, 3, 3).astype(np.float32)
    path = str(tmp_path / 'imagenet.pkl')
    with open(path, 'wb') as f:
        pickle.dump({'blobs': {'lr': 0.1, 'res2_0_branch2b_w': w2d}}, f, 2)
    CK.initialize_params_from_file(model, path, load_momentum=False)
    got = workspace.FetchBlob('gpu_0/res2_0_branch2b_w')
    assert got.shape == (128, 4, 1, 3, 3)
    np.testing.assert_array_equal(got[:, :, 0], w2d)
