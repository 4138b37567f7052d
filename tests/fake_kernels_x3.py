"""TEST-ONLY: a torch-CPU kernel stand-in (tests/fake_kernels.py, or resnext_oracle's with `groups`) whose GEMM wrappers
take the `precision` keyword of the real ones (vlfb.kernels), as a B200.COMPUTE 'tf32x3' net passes it.

The stand-in's products are exact in either precision, so `precision` only selects the dgrad weight transpose:
PREC_X3 stores w * scale unrounded (vlfb_weight_scale_transpose_multi), PREC_TF32 keeps the base's rounding."""
import inspect
import types

from vlfb import libvlfb as L

GEMMS = ('conv_fwd', 'conv_dgrad', 'conv_wgrad', 'conv_wgrad_det', 'matmul', 'matmul_det')


def _prec(precision):
    assert precision in (L.PREC_TF32, L.PREC_X3), precision


def _without_precision(f):
    """f with a trailing `precision` parameter (in its signature too: the launch audit binds the arguments by name)."""
    def g(*a, **kw):
        _prec(kw.pop('precision', L.PREC_TF32))
        return f(*a, **kw)
    sig = inspect.signature(f)
    g.__name__ = f.__name__
    g.__signature__ = sig.replace(parameters=list(sig.parameters.values()) + [
        inspect.Parameter('precision', inspect.Parameter.POSITIONAL_OR_KEYWORD, default=L.PREC_TF32)])
    return g


def _transpose(w, wt, s):
    co, ci = w.shape[0], w.shape[-1]
    t = w.reshape(co, -1, ci)
    if s is not None:
        t = t * s.view(-1, 1, 1)
    wt.copy_(t.permute(2, 1, 0).reshape(wt.shape))


def kernels(base):
    """A module with every function of `base` (copied now: patch `base` before calling this) and the GEMM wrappers and
    weight transposes taking `precision`."""
    mod = types.ModuleType(base.__name__ + '_x3')
    mod.__dict__.update(vars(base))
    for name in GEMMS:
        if hasattr(base, name):
            setattr(mod, name, _without_precision(getattr(base, name)))
    transpose = base.weight_transpose
    transpose_multi = base.weight_transpose_multi

    def weight_transpose(w, wt, scale=None, groups=1, precision=L.PREC_TF32):
        _prec(precision)
        if precision == L.PREC_TF32:
            return transpose(w, wt, scale) if groups == 1 else transpose(w, wt, scale, groups=groups)
        from vlfb.kernels import grouped_wt_slices
        for w_, wt_, s_ in grouped_wt_slices(w, wt, scale, groups):
            _transpose(w_, wt_, s_)

    def weight_transpose_multi(jobs, cache, precision=L.PREC_TF32):
        _prec(precision)
        if precision == L.PREC_TF32:
            return transpose_multi(jobs, cache)
        for w, wt, s in jobs:
            _transpose(w, wt, s)
    mod.weight_transpose, mod.weight_transpose_multi = weight_transpose, weight_transpose_multi
    return mod


def install(base):
    """Route vlfb.executor onto kernels(base) and the CPU device (fp64); returns that module."""
    import torch
    from vlfb import executor
    mod = kernels(base)
    executor.set_backend(mod, 'cpu', torch.float64)
    return mod
