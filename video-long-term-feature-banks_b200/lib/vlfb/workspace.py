"""Workspace shim: the subset of caffe2.python.workspace the reference's drivers use
(tools/train_net.py:74-75,152; lib/utils/metrics.py:521-560; lib/utils/checkpoints.py:376-381):
RunNetOnce / CreateNet / RunNet / FeedBlob / FetchBlob / HasBlob / ResetWorkspace.

One process drives ONE GPU (torchrun-style data parallelism) instead of Caffe2's
single-process-N-GPU model; blob names may carry the reference's 'gpu_{i}/' scope prefix,
which maps onto the local device.
"""
import re

import numpy as np
import torch

from . import executor as X
from .libvlfb import VlfbError

_SCOPE = re.compile(r'^gpu_\d+/')
STEM_PAD_L, STEM_PAD_R = 3, 5          # zero pixels around every row of a fed clip (conv1: kW = 7, pad 3, stride 2)
_INT_DTYPES = (torch.int32, torch.int64, torch.uint8, torch.bool, torch.int16, torch.int8)


def _unscoped(name):
    return _SCOPE.sub('', str(name))


class ParamStore(object):
    """All parameters live in flat fp32 buffers: P (master), Pt (TF32-rounded GEMM operand copy),
    G (gradients) and Mo (momentum).  Trainable parameters come first so that the gradient
    all-reduce and the fused SGD kernel run over contiguous ranges."""

    def __init__(self):
        self.chunks = []           # dict(P, Pt, G, Mo, size, n_nonfrozen)
        self.index = {}            # name -> (chunk, offset, numel, phys_shape, logical_shape, kind)
        self._trainable = set()
        self._mask = None

    def has(self, name):
        return name in self.index

    @staticmethod
    def _phys_shape(shape):
        shape = tuple(int(s) for s in shape)
        if len(shape) == 5:
            co, ci, kt, kh, kw = shape
            if ci == 3 and kw <= 8:
                return (co, kt, kh, 8, 4), 'stem'
            return (co, kt, kh, kw, ci), 'conv'
        return shape, 'plain'

    def add(self, specs, frozen):
        """specs: list of (name, logical_shape).  Allocates one chunk for the names not yet present."""
        new = [(n, s) for n, s in specs if n not in self.index]
        if not new:
            return
        new.sort(key=lambda ns: ns[0] in frozen)          # stable: non-frozen first
        off = 0
        entries = []
        n_nonfrozen = 0
        for name, shape in new:
            pshape, kind = self._phys_shape(shape)
            numel = int(np.prod(pshape))
            entries.append((name, off, numel, pshape, tuple(int(s) for s in shape), kind))
            off += (numel + 3) // 4 * 4
            if name not in frozen:
                n_nonfrozen = off
        ch = dict(P=torch.zeros(off, dtype=X.DTYPE, device=X.DEVICE),
                  Pt=torch.zeros(off, dtype=X.DTYPE, device=X.DEVICE), G=None, Mo=None, size=off,
                  n_nonfrozen=n_nonfrozen)
        self.chunks.append(ch)
        for name, o, numel, pshape, lshape, kind in entries:
            self.index[name] = (len(self.chunks) - 1, o, numel, pshape, lshape, kind)

    def _view(self, name, which):
        c, o, numel, pshape, _, _ = self.index[name]
        buf = self.chunks[c][which]
        return buf[o:o + numel].view(pshape)

    def phys(self, name):
        return self._view(name, 'P')

    def tf32(self, name):
        return self._view(name, 'Pt')

    def grad(self, name):
        return self._view(name, 'G')

    def momentum(self, name):
        self._ensure_state()
        return self._view(name, 'Mo')

    def logical_shape(self, name):
        return self.index[name][4]

    def _logical_of(self, pview, name):
        kind, lshape = self.index[name][5], self.index[name][4]
        if kind == 'conv':
            return pview.permute(0, 4, 1, 2, 3)
        if kind == 'stem':
            return pview[:, :, :, :lshape[4], :lshape[1]].permute(0, 4, 1, 2, 3)
        return pview

    def logical(self, name, which='P'):
        return self._logical_of(self._view(name, which), name)

    def refresh_tf32(self, name=None):
        if name is None:
            for ch in self.chunks:
                X.K.round_tf32(ch['P'], ch['Pt'])
        else:
            c, o, numel, _, _, _ = self.index[name]
            ch = self.chunks[c]
            X.K.round_tf32(ch['P'][o:o + numel], ch['Pt'][o:o + numel])

    def feed(self, name, arr):
        t = torch.as_tensor(np.asarray(arr)).to(X.DTYPE)
        dst = self.logical(name)
        assert tuple(t.shape) == tuple(dst.shape), 'shape mismatch feeding %s: %s vs %s' % (
            name, tuple(t.shape), tuple(dst.shape))
        if self.index[name][5] == 'stem':
            self._view(name, 'P').zero_()
        dst.copy_(t.to(X.DEVICE))
        self.refresh_tf32(name)

    def fetch(self, name, which='P'):
        t = self.logical(name, which).detach()
        a = t.cpu().contiguous().numpy()
        return a if t.is_cuda else a.copy()

    def stem_mask(self):
        if self._mask is None:
            m = torch.ones((8, 4), dtype=X.DTYPE)
            m[7, :] = 0
            m[:, 3] = 0
            self._mask = m.reshape(32).to(X.DEVICE)
        return self._mask

    # ---- training state
    def _ensure_state(self):
        for ch in self.chunks:
            if ch['G'] is None:
                ch['G'] = torch.zeros(ch['size'], dtype=X.DTYPE, device=X.DEVICE)
                ch['Mo'] = torch.zeros(ch['size'], dtype=X.DTYPE, device=X.DEVICE)

    def begin_step(self, trainable):
        self._ensure_state()
        self._trainable = set(trainable)
        for ch in self.chunks:
            if ch['n_nonfrozen']:
                X.K.fill(ch['G'][:ch['n_nonfrozen']], 0.0)

    def trainable(self, name):
        return name in self._trainable

    def scale_momentum(self, names, factor):
        self._ensure_state()
        for n in names:
            m = self._view(n, 'Mo').view(-1)
            X.K.axpby(m, factor, None, 0.0, m)

    def grad_ranges(self):
        """Contiguous gradient ranges to all-reduce: [(flat tensor view)]."""
        return [ch['G'][:ch['n_nonfrozen']] for ch in self.chunks if ch['n_nonfrozen'] and ch['G'] is not None]

    def sgd(self, trainable, lr, momentum, nesterov, wd_of):
        """Fused weight-decay + (Nesterov) momentum SGD over maximal contiguous runs of trainable
        parameters with equal weight decay (model_builder_video.py:375-388)."""
        tset = set(trainable)
        for ci, ch in enumerate(self.chunks):
            names = sorted([n for n, v in self.index.items() if v[0] == ci], key=lambda n: self.index[n][1])
            run = None            # (start, end, wd)
            runs = []
            for n in names:
                _, o, numel, _, _, _ = self.index[n]
                end = o + (numel + 3) // 4 * 4
                if n in tset:
                    wd = float(wd_of.get(n, 0.0))
                    if run is not None and run[1] == o and run[2] == wd:
                        run = (run[0], end, wd)
                    else:
                        if run is not None:
                            runs.append(run)
                        run = (o, end, wd)
                else:
                    if run is not None:
                        runs.append(run)
                        run = None
            if run is not None:
                runs.append(run)
            for s, e, wd in runs:
                X.K.sgd_nesterov(ch['P'][s:e], ch['G'][s:e], ch['Mo'][s:e], lr, momentum, wd, nesterov,
                                 ch['Pt'][s:e])
        self.sgd_launches = sum(1 for _ in [0])


class Workspace(object):
    def __init__(self):
        self.reset()

    def reset(self):
        self.blobs = {}
        self.rounded = set()
        self.params = ParamStore()
        self.nets = {}
        self.allreduce = None            # callable(ParamStore) installed by vlfb.dist
        self.reducer = None              # vlfb.dist.GradReducer (all-reduce overlapped with backward), built lazily
        self.overlap_allreduce = False
        self.dropout_enabled = True
        self.rng_seed = 2
        self.rng_offset = 0
        self.last_grads = {}
        self.input_cache = {}
        # asynchronous input queue (EnqueueBlobs): copy stream, staging slot, the batch waiting to be dequeued
        self.copy_stream = None
        self.queue_slot = 0
        self.queued = None
        self.slot_free = {}
        self.force_eager = False
        self.step = 0
        self._step_t = None
        # B200.ROI_CAPACITY (DESIGN.md 4.6): per-RoI input name -> (capacity C, suffix), registered by the nets that use
        # it; RoI-indexed blob name -> (C, suffix) (FetchBlob returns the live rows); suffix -> [device int32 live count,
        # host copy]; per-RoI input name -> the row count of its last feed
        self.roi_capacity = {}
        self.roi_blobs = {}
        self.roi_live = {}
        self.roi_fed = {}
        # B200.COMPUTE: float input name -> (compute mode, net name) of the nets that read it (executor.CompiledNet
        # _register_inputs); inputs of 'tf32x3' nets are stored unrounded
        self.input_compute = {}
        # B200.ITER_SIZE > 1: the training net whose iteration is under way (its gradients G hold a partial sum until the
        # boundary micro-step), else None
        self.open_iteration = None
        # B200.GPUS_PER_STEP (DESIGN.md 4.9): 'proposals{sfx}' name -> (v, b) of the packed training net that reads it;
        # name -> device int32 [v + 1] RoI row offsets of the virtual GPUs (fixed address, written in stream order by
        # every feed); name -> the (v, b) its last feed was checked for
        self.gpus_per_step = {}
        self.roi_segments = {}
        self.seg_fed = {}

    def begin_run(self):
        """Advance the device-side step counter (dropout masks of captured graphs depend on it)."""
        if X.DEVICE != 'cpu' or self._step_t is not None:
            self.step_tensor().fill_(self.step)
        self.step += 1

    def step_tensor(self):
        if self._step_t is None:
            self._step_t = torch.zeros(1, dtype=torch.int64, device=X.DEVICE)
        return self._step_t

    def next_rng(self, n):
        off = self.rng_offset
        self.rng_offset += (n + 3) // 4
        return self.rng_seed, off


_ws = Workspace()


def current():
    return _ws


def GlobalInit(args=None):
    return True


def ResetWorkspace():
    _ws.reset()
    return True


def Blobs():
    return list(_ws.blobs.keys()) + list(_ws.params.index.keys())


def HasBlob(name):
    name = _unscoped(name)
    return name in _ws.blobs or _ws.params.has(name)


_FILLS = ('ConstantFill', 'GaussianFill', 'MSRAFill', 'XavierFill', 'UniformFill')


def _fill_value(op, shape, gen):
    a = op.args
    if op.type == 'ConstantFill':
        return torch.full(shape, float(a.get('value', 0.0)))
    if op.type == 'GaussianFill':
        return torch.randn(shape, generator=gen) * float(a.get('std', 1.0)) + float(a.get('mean', 0.0))
    if op.type == 'MSRAFill':          # Caffe2: std = sqrt(2 / fan_out), fan_out = size / dim(1)
        fan_out = int(np.prod(shape)) // int(shape[1])
        return torch.randn(shape, generator=gen) * float(np.sqrt(2.0 / fan_out))
    if op.type == 'XavierFill':        # Caffe2: U(-s, s), s = sqrt(3 / fan_in), fan_in = size / dim(0)
        fan_in = int(np.prod(shape)) // int(shape[0])
        s = float(np.sqrt(3.0 / fan_in))
        return (torch.rand(shape, generator=gen) * 2 - 1) * s
    if op.type == 'UniformFill':
        lo, hi = float(a.get('min', 0.0)), float(a.get('max', 1.0))
        return torch.rand(shape, generator=gen) * (hi - lo) + lo
    raise NotImplementedError(op.type)


def RunNetOnce(net):
    """Execute a param_init_net: allocate + fill parameters (tools/train_net.py:74)."""
    from core.config import config as cfg
    model = getattr(net, '_model', None)
    params = (set(model.params) | set(getattr(model, 'computed_params', ()))) if model is not None else set()
    frozen = model.frozen_params if model is not None else set()
    specs, fills = [], []
    for op in net.ops:
        if op.type not in _FILLS:
            raise NotImplementedError('init op %s' % op.type)
        name = op.outputs[0]
        if name.endswith('_momentum'):
            continue                                   # momentum lives in the ParamStore
        shape = op.args.get('shape')
        if shape is None and op.inputs:
            shape = _ws.params.logical_shape(op.inputs[0]) if _ws.params.has(op.inputs[0]) else None
        if name in params:
            if not any(n == name for n, _ in specs) and not _ws.params.has(name):
                specs.append((name, tuple(shape)))
            fills.append((name, op, True))
        else:
            fills.append((name, op, False))
    _ws.params.add(specs, frozen)
    gen = torch.Generator().manual_seed(int(cfg.RNG_SEED))
    for name, op, is_param in fills:
        if is_param:
            shape = _ws.params.logical_shape(name)
            _ws.params.feed(name, _fill_value(op, tuple(shape), gen).numpy())
        else:
            shape = tuple(op.args.get('shape', [1]))
            _ws.blobs[name] = _fill_value(op, shape, gen).to(X.DTYPE).to(X.DEVICE)
    return True


def CreateNet(net, overwrite=False):
    """Lower the recorded net onto the kernels (tools/train_net.py:75)."""
    model = getattr(net, '_model', None)
    assert model is not None, 'CreateNet expects model.net of a vlfb CNNModelHelper'
    compiled = X.CompiledNet(model, _ws)
    _ws.nets[net.Proto().name] = compiled
    model._owner = compiled
    return True


def RunNet(name, num_iter=1):
    """One forward (+ backward + all-reduce + SGD for a training net) pass (tools/train_net.py:152)."""
    net = _ws.nets[str(name)]
    for _ in range(num_iter):
        _check_open_iteration(net)
        _dequeue_blobs()
        net.run()
    return True


def _check_open_iteration(net):
    """B200.ITER_SIZE: between the micro-steps of an iteration, G holds the gradients summed so far.  Another training
    net writes the same parameter store's G (and would update the parameters), so it may not run before the boundary;
    test nets only read the parameters and may."""
    owner = _ws.open_iteration
    if owner is not None and owner is not net and net.train:
        raise VlfbError('RunNet(%s): training net %s is at micro-step %d of %d of an iteration (B200.ITER_SIZE); '
                        'finish it before running another training net' % (net.name, owner.name, owner.micro,
                                                                           owner.iter_size))


def EnqueueBlobs(feed):
    """Asynchronous feeding: stands in for the reference's BlobsQueue + DequeueBlobs pair (dataloader.py:278-290,
    model_builder_video.py add_inputs).  `feed` maps blob names to (pinned) host tensors of the NEXT batch; the
    host-to-device copies run on a side stream into one of two staging slots, i.e. behind the step that is
    currently executing, and the next RunNet dequeues them (layout conversion + TF32 rounding into the static
    input buffers) before it starts.  One batch can be queued at a time."""
    ws = _ws
    if X.DEVICE == 'cpu':
        for name, arr in feed.items():
            FeedBlob(name, arr)
        return True
    assert ws.queued is None, 'EnqueueBlobs: the previous batch has not been consumed by RunNet yet'
    segs = dict((_unscoped(n), _segment_offsets(_unscoped(n), a)) for n, a in feed.items())    # checked on the host
    segs = dict((n, o) for n, o in segs.items() if o is not None)
    if ws.copy_stream is None:
        ws.copy_stream = torch.cuda.Stream()
    slot = ws.queue_slot
    ws.queue_slot ^= 1
    main = torch.cuda.current_stream()
    free = ws.slot_free.get(slot)
    if free is not None:
        ws.copy_stream.wait_event(free)            # the conversion kernels that read this slot have finished
    staged = {}
    with torch.cuda.stream(ws.copy_stream):
        for name, arr in feed.items():
            src = arr if isinstance(arr, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(arr))
            is_int = src.dtype in _INT_DTYPES
            shape = tuple(src.shape)
            cap = _roi_rows(_unscoped(name), shape)
            if cap is not None:
                shape = (cap,) + shape[1:]              # a per-RoI input: the slot keeps its C-row shape and address
            st = _static('%s/stage%d' % (_unscoped(name), slot), shape, torch.int32 if is_int else X.DTYPE)
            if cap is not None:
                st = st[:src.shape[0]]
            st.copy_(src, non_blocking=True)
            staged[_unscoped(name)] = st
        ev = torch.cuda.Event()
        ev.record(ws.copy_stream)
    ws.queued = (slot, staged, ev, segs)
    del main
    return True


def _dequeue_blobs():
    ws = _ws
    if ws.queued is None:
        return
    slot, staged, ev, segs = ws.queued
    ws.queued = None
    torch.cuda.current_stream().wait_event(ev)
    for name, st in staged.items():
        _feed_activation(name, st)
    for name, offs in segs.items():
        _set_segments(name, offs)
    done = torch.cuda.Event()
    done.record(torch.cuda.current_stream())
    ws.slot_free[slot] = done


def _static(key, shape, dtype):
    """Persistent device buffer: the address is stable while the shape is unchanged (CUDA-graph replay
    and allocation-free feeding)."""
    t = _ws.input_cache.get(key)
    if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
        t = torch.empty(tuple(shape), dtype=dtype, device=X.DEVICE)
        _ws.input_cache[key] = t
    return t


def _roi_rows(name, shape):
    """Capacity C when `name` is a per-RoI input of a B200.ROI_CAPACITY net (None otherwise), after checking that the
    `shape[0]` rows fed fit it."""
    ent = _ws.roi_capacity.get(name)
    if ent is None:
        return None
    cap = ent[0]
    r = int(shape[0]) if len(shape) else 0
    if not 1 <= r <= cap:
        raise VlfbError('%s: %d RoI rows fed; B200.ROI_CAPACITY = %d holds 1 to %d' % (name, r, cap, cap))
    return cap


def _segment_offsets(name, arr):
    """B200.GPUS_PER_STEP: for a 'proposals' input of a packed training net, check the fed RoIs against the packed
    batch's rules -- batch indices (column 0) in [0, v b) and not decreasing -- and return the v + 1 row offsets of the
    virtual GPUs' RoIs (virtual GPU j = batch index // b).  None for any other input."""
    ent = _ws.gpus_per_step.get(name)
    if ent is None:
        return None
    v, b = ent
    a = arr.detach().cpu().numpy() if isinstance(arr, torch.Tensor) else np.asarray(arr)
    if a.ndim != 2 or a.shape[1] < 1:
        raise VlfbError('%s: RoIs of shape %s; B200.GPUS_PER_STEP expects [R, 5] rows (batch index first)'
                        % (name, tuple(a.shape)))
    idx = a[:, 0]
    if idx.size and (not np.all(idx == np.floor(idx)) or idx.min() < 0 or idx.max() >= v * b):
        raise VlfbError('%s: batch indices must be integers in [0, %d) for B200.GPUS_PER_STEP = %d virtual GPUs of %d '
                        'clips' % (name, v * b, v, b))
    if idx.size > 1 and np.any(np.diff(idx) < 0):
        raise VlfbError('%s: batch indices decrease; a packed batch lists virtual GPU j\'s RoIs (batch index in [j b, '
                        '(j+1) b)) before those of virtual GPU j + 1' % name)
    return np.searchsorted(idx.astype(np.int64), np.arange(v + 1) * b, side='left').astype(np.int32)


def _set_segments(name, offs):
    """Write the row offsets of the virtual GPUs' RoIs into the input's fixed device buffer, in stream order (a captured
    graph reads each replay's offsets), and record which (v, b) the feed was checked for."""
    buf = _ws.roi_segments.get(name)
    if buf is None or buf.numel() != len(offs):
        buf = _ws.roi_segments[name] = torch.zeros(len(offs), dtype=torch.int32, device=X.DEVICE)
    buf.copy_(torch.from_numpy(offs))
    _ws.seg_fed[name] = _ws.gpus_per_step[name]


def set_live_rows(name, rows):
    """Record that per-RoI input `name` was fed `rows` live rows: the host copy, and the device count the kernels read,
    written in stream order behind the feed."""
    sfx = _ws.roi_capacity[name][1]
    ent = _ws.roi_live.get(sfx)
    if ent is None:
        ent = _ws.roi_live[sfx] = [torch.zeros(1, dtype=torch.int32, device=X.DEVICE), 0]
    ent[0].fill_(int(rows))
    ent[1] = int(rows)
    _ws.roi_fed[name] = int(rows)


def _input_buffer(name, src, dtype):
    """The static device buffer of input `name` holding `src`.  A per-RoI input of a B200.ROI_CAPACITY net gets C rows:
    the r fed rows, then rows [r, C) rewritten with padding at every feed (labels -1, the sigmoid loss's ignore value;
    anything else 0), so that its shape and address never change and no padded row holds stale or uninitialised data."""
    cap = _roi_rows(name, tuple(src.shape))
    if cap is None:
        dst = _static(name, src.shape, dtype)
        dst.copy_(src, non_blocking=True)
        return dst
    r = int(src.shape[0])
    dst = _static(name, (cap,) + tuple(src.shape[1:]), dtype)
    dst[:r].copy_(src, non_blocking=True)
    dst[r:].fill_(-1 if name.startswith('labels') else 0)
    set_live_rows(name, r)
    return dst


def feeds_unrounded(name):
    """True when input `name` is read by B200.COMPUTE 'tf32x3' nets: its feeds are stored without the TF32 rounding."""
    return _ws.input_compute.get(name, ('tf32',))[0] == 'tf32x3'


def _feed_activation(name, arr):
    src = arr if isinstance(arr, torch.Tensor) else torch.as_tensor(np.ascontiguousarray(arr))
    rnd = not feeds_unrounded(name)
    if src.dtype in _INT_DTYPES:
        dst = _input_buffer(name, src, torch.int32)
        _ws.blobs[name] = dst
        _ws.rounded.discard(name)
        return
    if src.dim() == 5:
        n, c = src.shape[0], src.shape[1]
        inner = src.shape[2] * src.shape[3] * src.shape[4]
        cpad = 4 if c == 3 else c
        if src.is_cuda and src.dtype == X.DTYPE:
            stage = src                                           # already staged on the device (EnqueueBlobs)
        else:
            stage = _static(name + '/ncthw', src.shape, X.DTYPE)
            stage.copy_(src, non_blocking=True)                   # H2D (async from pinned memory)
        t_, h_, w_ = int(src.shape[2]), int(src.shape[3]), int(src.shape[4])
        if c == 3 and w_ % 4 == 0 and X.DEVICE != 'cpu':
            # the clip feeds conv1 only: rows are stored with STEM_PAD_L zero pixels on the left and zero pixels up to
            # the pitch on the right, so that a filter row's 8-pixel window of ANY output position is 128 contiguous
            # in-bounds bytes and the stem operand can be staged by TMA (csrc/gemm_tc.cu make_tmap_stem)
            pitch = (STEM_PAD_L + w_ + STEM_PAD_R + 3) // 4 * 4
            key = name + '/padded'
            buf = _ws.input_cache.get(key)
            if buf is None or tuple(buf.shape) != (n, t_, h_, pitch, cpad):
                buf = torch.zeros((n, t_, h_, pitch, cpad), dtype=X.DTYPE, device=X.DEVICE)     # pads stay zero
                _ws.input_cache[key] = buf
            X.K.nc_to_cl(stage, buf, n, c, inner, cpad, tf32_out=rnd, width=w_, pitch=pitch, left=STEM_PAD_L)
            _ws.blobs[name] = buf[:, :, :, STEM_PAD_L:STEM_PAD_L + w_, :].permute(0, 4, 1, 2, 3)
            _mark_rounded(name, rnd)
            return
        p = _static(name, (n, t_, h_, w_, cpad), X.DTYPE)
        X.K.nc_to_cl(stage, p, n, c, inner, cpad, tf32_out=rnd)   # reference NCTHW blob -> NDHWC (+pad 3->4), TF32-rounded
        _ws.blobs[name] = p.permute(0, 4, 1, 2, 3)
        _mark_rounded(name, rnd)
        return
    dst = _input_buffer(name, src, X.DTYPE)
    bank_companion(name, dst)
    if rnd and dst.dim() >= 2 and dst.shape[-1] >= 64:            # feature banks are GEMM operands
        X.K.round_tf32(dst.view(-1), dst.view(-1))
        _ws.rounded.add(name)
    else:
        _ws.rounded.discard(name)
    _ws.blobs[name] = dst


def _mark_rounded(name, rounded):
    if rounded:
        _ws.rounded.add(name)
    else:
        _ws.rounded.discard(name)


def bank_companion(name, dst):
    """B200.LFB_DTYPE 'bf16': keep a bf16 copy of a fed feature bank ('lfb*' blobs, rows of 2048 / 4096 features) under
    '<name>@bf16' -- the operand of the folded inference FBO's bank scan (executor.FboFoldStep), half the HBM bytes per
    pass.  The fp32 blob stays (the as-written / training lowerings read it).  Any other setting drops a stale copy."""
    from core.config import config as cfg
    key = name + '@bf16'
    if (cfg.B200.get('LFB_DTYPE', 'f32') == 'bf16' and name.startswith('lfb') and dst.dim() == 3
            and int(dst.shape[-1]) in (2048, 4096)):
        comp = _static(key, dst.shape, torch.bfloat16)
        X.K.cast_bf16(dst.view(-1), comp.view(-1))
        _ws.blobs[key] = comp
    else:
        _ws.blobs.pop(key, None)


def FeedBlob(name, arr, device_option=None):
    name = _unscoped(name)
    if _ws.params.has(name):
        _ws.params.feed(name, arr)
        return True
    if name.endswith('_momentum') and _ws.params.has(name[:-len('_momentum')]):
        base = name[:-len('_momentum')]
        _ws.params._ensure_state()
        _ws.params.logical(base, 'Mo').copy_(torch.as_tensor(np.asarray(arr)).to(X.DTYPE).to(X.DEVICE))
        return True
    offs = _segment_offsets(name, arr)                 # checked before anything is written
    if np.ndim(arr) == 0 or name in ('lr', 'weight_decay', 'weight_decay_bn', 'ONE'):
        v = torch.as_tensor(np.asarray(arr).reshape(-1)).to(X.DTYPE)
        cur = _ws.blobs.get(name)
        if isinstance(cur, torch.Tensor) and cur.shape == v.shape:
            cur.copy_(v)                                           # in place: captured graphs read this address
        else:
            _ws.blobs[name] = v.to(X.DEVICE)
        return True
    _feed_activation(name, arr)
    if offs is not None:
        _set_segments(name, offs)                      # only once the feed itself has landed
    return True


class _PendingFetch(object):
    """Handle returned by FetchBlobAsync: .get() waits for the device->host copy and returns the numpy value."""

    def __init__(self, host, event, scalar, rows=None):
        self._host, self._event, self._scalar, self._rows = host, event, scalar, rows

    def ready(self):
        return self._event is None or self._event.query()

    def get(self):
        if self._event is not None:
            self._event.synchronize()
        a = self._host if isinstance(self._host, np.ndarray) else self._host.numpy().copy()
        if self._rows is not None:
            a = a[:self._rows]
        return a.reshape(()) if (self._scalar and a.size == 1) else a


def FetchBlobAsync(name):
    """Non-blocking FetchBlob for small activation blobs (loss, pred, metrics): the device->host copy is enqueued on
    the current stream behind the work already submitted, into one of four pinned staging buffers per blob; the
    returned handle's .get() waits for that copy only.  A training loop reads step i's loss after it has launched
    step i+1, so the device never idles behind the host (the reference's FetchBlob after every RunNet,
    tools/train_net.py:152-160, serialises the two)."""
    name = _unscoped(name)
    scalar = name in ('loss', 'lr') or name.startswith('loss')
    if X.DEVICE == 'cpu' or _ws.params.has(name):
        return _PendingFetch(np.asarray(FetchBlob(name)), None, scalar)
    t = _ws.blobs[name]
    assert isinstance(t, torch.Tensor), 'FetchBlobAsync: %s is not a tensor blob' % name
    ring = _ws.input_cache.setdefault('fetch_ring/' + name, [[], 0])
    if len(ring[0]) < 4 or tuple(ring[0][0].shape) != tuple(t.shape):
        if ring[0] and tuple(ring[0][0].shape) != tuple(t.shape):
            ring[0], ring[1] = [], 0
        ring[0].append(torch.empty(tuple(t.shape), dtype=t.dtype).pin_memory())
        host = ring[0][-1]
    else:
        host = ring[0][ring[1] % 4]
    ring[1] += 1
    host.copy_(t, non_blocking=True)         # strided logical views are copied element-wise: logical layout on the host
    ev = torch.cuda.Event()
    ev.record(torch.cuda.current_stream())
    return _PendingFetch(host, ev, scalar, live_rows(name, t))


def live_rows(name, t):
    """Number of live rows of blob `name` (tensor t) when it is RoI-indexed in a B200.ROI_CAPACITY net, else None."""
    ent = _ws.roi_blobs.get(name)
    if ent is None or t.dim() == 0 or int(t.shape[0]) != ent[0] or ent[1] not in _ws.roi_live:
        return None
    return _ws.roi_live[ent[1]][1]


def FetchBlob(name):
    name = _unscoped(name)
    if _ws.params.has(name):
        return _ws.params.fetch(name)
    if name.endswith('_momentum') and _ws.params.has(name[:-len('_momentum')]):
        _ws.params._ensure_state()
        return _ws.params.fetch(name[:-len('_momentum')], 'Mo')
    if name.endswith('_grad') and _ws.params.has(name[:-len('_grad')]):
        return _ws.params.fetch(name[:-len('_grad')], 'G')
    t = _ws.blobs[name]
    if isinstance(t, tuple):
        return np.array(t, dtype=np.int64)
    if t.dim() == 5 and t.shape[1] == 4 and name.startswith('data'):
        t = t[:, :3]
    rows = live_rows(name, t)
    if rows is not None:
        t = t[:rows]
    a = t.detach().cpu().contiguous().numpy()
    if not t.is_cuda:
        a = a.copy()              # the CPU test engine would otherwise hand out a view of a reusable input buffer
    if name in ('loss', 'lr') or a.size == 1 and name.startswith('loss'):
        return a.reshape(()) if a.size == 1 else a
    return a
