"""One-process-per-GPU data parallelism: NCCL all-reduce (sum) of the flat gradient buffers
and the initial parameter broadcast.  Replaces Caffe2's per-parameter NCCLAllreduce ops
(SURVEY.md section 2 row 8) and checkpoints.broadcast_parameters (lib/utils/checkpoints.py:386-407).

torch.distributed is plumbing only (NCCL communicator + stream handling); on CPU test
runs the same code path uses the gloo backend.
"""
import os

import torch
import torch.distributed as dist

BUCKET_ELEMS = 8 * 1024 * 1024        # 32 MB fp32 buckets: large enough to saturate NVLink 5


def init_from_env(backend=None):
    """Initialise the default process group from torchrun's environment.  Returns (rank, world)."""
    world = int(os.environ.get('WORLD_SIZE', '1'))
    rank = int(os.environ.get('RANK', '0'))
    if world > 1 and not dist.is_initialized():
        if backend is None:
            backend = 'nccl' if torch.cuda.is_available() else 'gloo'
        if backend == 'nccl':
            local = int(os.environ.get('LOCAL_RANK', '0'))
            torch.cuda.set_device(local)
            dist.init_process_group(backend=backend, device_id=torch.device('cuda', local))
        else:
            dist.init_process_group(backend=backend)
    return rank, world


def shutdown(timeout_s=20.0):
    """Leave the process group.  The captured training step holds NCCL kernels (overlapped all-reduce inside the graph) and
    ncclCommDestroy waits for every CUDA graph that captured the communicator: the graphs are released first (the nets of
    the workspace are dropped), and the teardown runs under a watchdog, so that a benchmark that has printed its line
    never sits in destroy_process_group().  Returns False if the teardown had to be abandoned."""
    if not dist.is_initialized():
        return True
    import gc
    import threading
    done = []

    def teardown():
        try:
            import torch
            from . import workspace
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            workspace.ResetWorkspace()          # CompiledNet._graphs -> CUDAGraph destructors
            gc.collect()
            if torch.cuda.is_available():
                torch.cuda.synchronize()
            dist.destroy_process_group()
        except Exception as exc:                 # a failing teardown must not turn a finished run into an error
            import sys
            sys.stderr.write('vlfb.dist.shutdown: %r\n' % (exc,))
        done.append(True)

    th = threading.Thread(target=teardown, daemon=True)
    th.start()
    th.join(timeout_s)
    return bool(done)


def world_size():
    return dist.get_world_size() if dist.is_initialized() else 1


def allreduce_grads(store):
    """Sum the gradient ranges across ranks, bucket by bucket (async, then one wait)."""
    if world_size() == 1:
        return 0
    handles = []
    for flat in store.grad_ranges():
        for s in range(0, flat.numel(), BUCKET_ELEMS):
            handles.append(dist.all_reduce(flat[s:s + BUCKET_ELEMS], op=dist.ReduceOp.SUM, async_op=True))
    for h in handles:
        h.wait()
    return len(handles)


class GradReducer(object):
    """Bucketed gradient all-reduce OVERLAPPED with backward (SURVEY 8e; the reference's per-parameter NCCLAllreduce
    ops are scheduled by Caffe2's dag executor as their inputs become ready, model_builder_video.py:147-157).

    The flat gradient buffer is cut into buckets of BUCKET_ELEMS; the executor reports every parameter whose gradient
    is complete (`param_done`) and a bucket's all-reduce is issued -- asynchronously, on the communicator's stream, as
    soon as its last parameter is -- while the rest of backward keeps the SMs busy; `finish` issues what is left and
    makes the compute stream wait.  Parameters are laid out in forward order and backward visits them in reverse, so the
    buckets complete from the end of the buffer towards its start.  Stream-ordered only (no host synchronisation): the
    whole step, collectives included, can be captured into ONE CUDA graph."""

    def __init__(self, store):
        self.store = store
        self.buckets = []            # (chunk index, start, end)
        self.of_param = {}           # name -> bucket ids it overlaps
        for ci, ch in enumerate(store.chunks):
            n = ch['n_nonfrozen']
            first = len(self.buckets)
            for s in range(0, n, BUCKET_ELEMS):
                self.buckets.append((ci, s, min(n, s + BUCKET_ELEMS)))
            for name, (c, off, numel, _, _, _) in store.index.items():
                if c != ci or off >= n:
                    continue
                lo, hi = off // BUCKET_ELEMS, (off + numel - 1) // BUCKET_ELEMS
                self.of_param[name] = [first + b for b in range(lo, hi + 1)]
        self.total = [0] * len(self.buckets)
        for bs in self.of_param.values():
            for b in bs:
                self.total[b] += 1
        self.remaining, self.launched, self.handles = [], [], []

    def begin(self):
        self.remaining = list(self.total)
        self.launched = [False] * len(self.buckets)
        self.handles = []

    def _launch(self, b):
        ci, s, e = self.buckets[b]
        self.launched[b] = True
        self.handles.append(dist.all_reduce(self.store.chunks[ci]['G'][s:e], op=dist.ReduceOp.SUM, async_op=True))

    def param_done(self, name):
        for b in self.of_param.get(name, ()):
            self.remaining[b] -= 1
            if self.remaining[b] == 0 and not self.launched[b]:
                self._launch(b)

    def finish(self):
        for b in range(len(self.buckets)):
            if not self.launched[b]:
                self._launch(b)
        for h in self.handles:
            h.wait()
        n, self.handles = len(self.handles), []
        return n


def broadcast_params(store, src=0):
    """Rank `src`'s parameters (and momentum, when allocated) become everyone's."""
    if world_size() == 1:
        return
    for ch in store.chunks:
        dist.broadcast(ch['P'], src)
        dist.broadcast(ch['Pt'], src)
        if ch['Mo'] is not None:
            dist.broadcast(ch['Mo'], src)


def install(ws):
    """Hook the gradient all-reduce into workspace.RunNet for training nets: overlapped with backward (GradReducer,
    B200.OVERLAP_ALLREDUCE / VLFB_OVERLAP=0 to disable) or, as a fallback, after it (allreduce_grads)."""
    ws.allreduce = allreduce_grads if world_size() > 1 else None
    ws.reducer = None
    ws.overlap_allreduce = world_size() > 1 and os.environ.get('VLFB_OVERLAP', '1') != '0' 
