"""B200.ROI_CAPACITY on the fp64 CPU engine (tests/fake_kernels.py, with the live row count added by
tests/fake_live_rows.py): a net built at C RoI rows and fed r <= C rows must compute what a C = 0 net fed the same r rows
computes (loss, the live rows of the RoI-indexed blobs, every parameter gradient), hold only finite values in every
padded row -- even when every buffer starts as NaN -- and reject what it cannot run."""
import numpy as np
import pytest
import torch

import harness as H

TINY = ['NUM_GPUS', 1, 'TRAIN.BATCH_SIZE', 2, 'TRAIN.CROP_SIZE', 64, 'TRAIN.VIDEO_LENGTH', 8,
        'TEST.BATCH_SIZE', 2, 'TEST.CROP_SIZE', 64, 'TEST.VIDEO_LENGTH', 8, 'LFB.WINDOW_SIZE', 4,
        'TRAIN.DROPOUT_RATE', 0.0, 'FBO_NL.INPUT_DROPOUT_ON', False, 'FBO_NL.LFB_DROPOUT_ON', False]
YAML = 'ava_r50_lfb_nl.yaml'
CAP = 8
ROWS = (3, 8, 1)
PER_ROI = ('proposals', 'labels', 'original_boxes', 'metadata', 'lfb')


@pytest.fixture
def fake(monkeypatch):
    """The CPU engine, with every activation the executor allocates starting as NaN (ints as garbage): a padded row that a
    kernel forgot to write would poison the comparison below."""
    import fake_kernels
    import fake_live_rows
    from vlfb import executor as X, workspace
    fake_kernels.install()
    fake_live_rows.install(monkeypatch)
    workspace.ResetWorkspace()

    def poisoned(t):
        return t.fill_(float('nan')) if t.is_floating_point() else t.fill_(-12345)
    empty, empty_like = X.empty, X.empty_like_strided
    monkeypatch.setattr(X, 'empty', lambda shape, dtype=None: poisoned(empty(shape, dtype)))
    monkeypatch.setattr(X, 'empty_like_strided', lambda t: poisoned(empty_like(t)))
    yield fake_kernels
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


def _inputs(ocfg):
    from oracle import model as OM
    inputs = OM.make_inputs(ocfg, n_clips=2, rois_per_clip=CAP // 2, crop=64, frames=8)
    g = torch.Generator().manual_seed(5)
    inputs['metadata'] = torch.rand((CAP, 4), generator=g) * 100
    inputs['original_boxes'] = torch.rand((CAP, 4), generator=g)
    return inputs


def _feed(inputs, sfx, r):
    from vlfb import workspace
    for name, t in inputs.items():
        t = t[:r] if name in PER_ROI else t
        workspace.FeedBlob('gpu_0/{}{}'.format(name, sfx), t.double().numpy() if t.dtype == torch.float32 else t.numpy())


def _build(cap, split, train, lfb_infer_only=False, extra=()):
    from vlfb import workspace
    H.setup_cfg(YAML, TINY + ['B200.ROI_CAPACITY', cap] + list(extra))
    workspace.ResetWorkspace()
    model, sfx = H.build(split, train, lfb_infer_only=lfb_infer_only)
    return model, sfx


def _poison_inputs(sfx, inputs):
    """Pre-create the C-row input buffers holding NaN / garbage, so that the first feed finds them dirty."""
    from vlfb import executor as X, workspace
    ws = workspace.current()
    for name in PER_ROI:
        if name not in inputs or name + sfx not in ws.roi_capacity:
            continue
        t = inputs[name]
        is_int = not t.is_floating_point()
        shape = (CAP,) + tuple(t.shape[1:])
        ws.input_cache[name + sfx] = (torch.full(shape, 77, dtype=torch.int32) if is_int else
                                      torch.full(shape, float('nan'), dtype=X.DTYPE))


def _run(cap, split, train, blobs, lfb_infer_only=False):
    """Per r of ROWS: loss, the named blobs and every parameter gradient after one forward (+ backward) pass."""
    from oracle import model as OM
    from vlfb import workspace
    ocfg = H.oracle_cfg(YAML, TINY)
    params = OM.make_params(ocfg, seed=2, split=split, lfb_infer_only=lfb_infer_only) if not train else \
        OM.make_params(ocfg, seed=2)
    inputs = _inputs(ocfg)
    model, sfx = _build(cap, split, train, lfb_infer_only)
    net = workspace.current().nets[model.net.Proto().name]
    net.update_ops = []                                           # gradients of the same initial state every step
    H.feed_params(dict((k, v) for k, v in params.items() if workspace.HasBlob(k)))
    if cap:
        assert net.roi_capacity == cap and 'proposals' + sfx in net.roi_inputs
        _poison_inputs(sfx, inputs)
    out = []
    for r in ROWS:
        _feed(inputs, sfx, r)
        workspace.RunNet(model.net.Proto().name)
        res = dict((b, workspace.FetchBlob('gpu_0/' + b.format(sfx=sfx))) for b in blobs)
        if train:
            res['loss'] = workspace.FetchBlob('gpu_0/loss')
            res['grads'] = dict((n, workspace.FetchBlob('gpu_0/' + n + '_grad')) for n in model.TrainableParams())
        if cap:
            ws = workspace.current()
            for name, t in ws.blobs.items():                      # every buffer, padded rows included
                if isinstance(t, torch.Tensor) and t.is_floating_point():
                    assert torch.isfinite(t).all(), (r, name)
            for ch in ws.params.chunks:
                assert ch['G'] is None or torch.isfinite(ch['G']).all()
        out.append(res)
    return out


def _close(a, b, tol=1e-10):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    assert a.shape == b.shape, (a.shape, b.shape)
    assert np.isfinite(a).all()
    return float(np.abs(a - b).max(initial=0.0)) <= tol * max(float(np.abs(b).max(initial=0.0)), 1e-5)


def _compare(blobs, split, train, lfb_infer_only=False):
    ref = _run(0, split, train, blobs, lfb_infer_only)
    got = _run(CAP, split, train, blobs, lfb_infer_only)
    for r, a, b in zip(ROWS, got, ref):
        for name in blobs:
            assert a[name].shape[0] == r, (name, a[name].shape)
            assert _close(a[name], b[name]), (r, name)
        if train:
            assert _close(a['loss'], b['loss']), r
            assert sorted(a['grads']) == sorted(b['grads'])
            for n in b['grads']:
                assert _close(a['grads'][n], b['grads'][n]), (r, n)


def test_training_net_at_capacity_matches_exact_rows(fake):
    _compare(['box_pooled', 'pool5', 'pred', 'prob', 'labels{sfx}', 'proposals{sfx}'], 'train', True)


def test_test_net_at_capacity_matches_exact_rows(fake):
    _compare(['box_pooled', 'lfb_nl0_affinity_prob', 'pool5', 'pred', 'prob'], 'val', False)


def test_lfb_infer_only_net_at_capacity_matches_exact_rows(fake):
    _compare(['box_pooled', 'metadata{sfx}'], 'val', False, lfb_infer_only=True)


def test_fetch_blob_async_returns_the_live_rows(fake):
    from oracle import model as OM
    from vlfb import workspace
    ocfg = H.oracle_cfg(YAML, TINY)
    model, sfx = _build(CAP, 'train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    _feed(_inputs(ocfg), sfx, 5)
    workspace.RunNet(model.net.Proto().name)
    for name in ('pred', 'loss', 'labels' + sfx):
        a, b = workspace.FetchBlob('gpu_0/' + name), workspace.FetchBlobAsync('gpu_0/' + name).get()
        assert np.array_equal(a, b)
    assert workspace.FetchBlob('gpu_0/pred').shape[0] == 5
    assert workspace.current().blobs['pred'].shape[0] == CAP
    assert workspace.FetchBlob('gpu_0/conv1_w').shape[0] == 64            # parameters are never sliced


def test_error_cases(fake):
    from oracle import model as OM
    from vlfb import workspace
    from vlfb.libvlfb import VlfbError
    ocfg = H.oracle_cfg(YAML, TINY)
    inputs = _inputs(ocfg)
    model, sfx = _build(CAP, 'train', True)
    H.feed_params(OM.make_params(ocfg, seed=2))
    name = 'gpu_0/proposals' + sfx
    big = np.zeros((CAP + 1, 5))
    with pytest.raises(VlfbError, match='proposals' + sfx):
        workspace.FeedBlob(name, big)                                      # r > C
    with pytest.raises(VlfbError, match='proposals' + sfx):
        workspace.FeedBlob(name, np.zeros((0, 5)))                         # r = 0
    _feed(inputs, sfx, 4)
    workspace.FeedBlob('gpu_0/labels' + sfx, inputs['labels'][:3].numpy())
    with pytest.raises(VlfbError, match='labels' + sfx):
        workspace.RunNet(model.net.Proto().name)                           # one step, two RoI counts
    _feed(inputs, sfx, 4)
    workspace.RunNet(model.net.Proto().name)                               # consistent again: runs
    # a softmax loss averages over all rows, padding included
    with pytest.raises(VlfbError, match='SoftmaxWithLoss'):
        _build(CAP, 'train', True, extra=['MODEL.MULTI_LABEL', False])


def test_default_capacity_is_off_and_registers_nothing(fake):
    from core.config import config as cfg
    from vlfb import workspace
    model, sfx = _build(0, 'train', True)
    assert cfg.B200.ROI_CAPACITY == 0
    net = workspace.current().nets[model.net.Proto().name]
    assert net.roi_capacity == 0 and not net.roi_blobs and not workspace.current().roi_capacity


def test_device_lfb_feed_pads_the_index_table(fake):
    from datasets.lfb_bank import DeviceLfb
    from vlfb import workspace
    model, sfx = _build(CAP, 'val', False)
    dim = 2048
    bank = DeviceLfb({0: {s: [np.full(dim, s + 1.0)] for s in range(6)}}, dim)
    ws = workspace.current()
    L = 8
    table = np.arange(3 * L, dtype=np.int32).reshape(3, L) % 6
    ws.input_cache['lfb' + sfx] = torch.full((CAP, L, dim), float('nan'), dtype=torch.float64)
    dst = bank.feed('gpu_0/lfb' + sfx, table)
    assert tuple(dst.shape) == (CAP, L, dim) and ws.roi_fed['lfb' + sfx] == 3
    assert torch.equal(dst[3:], torch.zeros_like(dst[3:]))
    assert torch.equal(dst[:3, :, 0], torch.as_tensor(table + 1.0, dtype=dst.dtype))
    assert workspace.FetchBlob('gpu_0/lfb' + sfx).shape == (3, L, dim)
    assert int(ws.roi_live[sfx][0]) == 3
