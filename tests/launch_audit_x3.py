"""Launch audit (tests/launch_audit.py) of B200.COMPUTE 'tf32x3' nets: the same audit, with the split-TF32 GEMM calls
(precision = PREC_X3) held to what they compute.  For such a call
  * the value reference reads the operands as they are (the tensor core splits them; it does not truncate them),
  * the elementwise bound is gemm_x3.tau_x3(K) instead of tau(K),
  * the TF32-exactness check of the operands does not apply (a 'tf32x3' net rounds nothing),
and the dgrad weight transpose of a PREC_X3 call is held bit for bit to the unrounded w * scale.  Every other call is
audited exactly as launch_audit.py audits it.

    python tests/launch_audit_x3.py --net NAME --out FILE      (NAME: a net of NETS below)
"""
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import launch_audit as LA  # noqa: E402

X3 = ['B200.COMPUTE', 'tf32x3']
X3_TRAIN_WRAPPERS = LA.AVA_TRAIN_WRAPPERS - {'round_tf32'}
ROUNDING_WRAPPERS = ('round_tf32', 'add_tf32', 'relu_tf32', 'relu_bwd_tf32', 'add_relu_bwd_tf32')

# name -> (yaml, overrides, split, runs, wrappers the net must reach, extra settings), as launch_audit.NETS
NETS = {
    'ava_train_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + X3, 'train', 2, X3_TRAIN_WRAPPERS, {}),
    'ava_train_det_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + X3 + ['B200.DETERMINISTIC', True], 'train', 2,
                         {'conv_fwd', 'conv_dgrad', 'conv_wgrad_det', 'matmul_det', 'roi_align_bwd_det', 'sgd_nesterov'},
                         {}),
    'ava_train_capacity_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + X3 + ['B200.ROI_CAPACITY', 8], 'train', 2,
                              X3_TRAIN_WRAPPERS, {}),
    'ava_val_fold_f32_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + X3, 'val', 1, {'conv_fwd', 'fbo_bank_scan', 'roi_align_fwd'},
                            {}),
    'ava_lfb_infer_only_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + X3, 'lfb_infer_only', 1, {'conv_fwd', 'roi_align_fwd'},
                              {}),
    'charades_softmax_train_x3': ('charades_r50_lfb_nl.yaml', LA.TINY + X3 + ['MODEL.NUM_CLASSES', 157,
                                                                               'MODEL.MULTI_LABEL', False],
                                  'train', 2, {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'matmul', 'softmax_ce_fwd',
                                               'softmax_ce_bwd', 'sgd_nesterov'}, {}),
    'resnext_bn_train_x3': ('ava_r50_lfb_nl.yaml', LA.TINY + LA.RESNEXT + X3, 'train', 2,
                            {'conv_fwd', 'conv_dgrad', 'conv_wgrad', 'spatial_bn_fwd', 'spatial_bn_bwd', 'sgd_nesterov'},
                            {'grouped': True}),
}


def is_x3(b):
    """True for a split-TF32 call (the wrapper's precision = PREC_X3)."""
    from vlfb import libvlfb as L
    return b.get('precision') == L.PREC_X3


def install(patch=setattr):
    """Extend launch_audit in place (patch(obj, name, value): setattr, or a test's monkeypatch.setattr)."""
    gemm_operand, gemm_bound, wt_multi = LA._gemm_operand, LA._gemm_bound, LA.REF['weight_transpose_multi']
    base = LA.Audit

    def operand(c, t):
        return t if is_x3(c.b) else gemm_operand(c, t)

    def bound(c, mag, K):
        if c.engine == 'tcgen05' and is_x3(c.b):
            import gemm_x3
            return mag * (gemm_x3.tau_x3(K) / LA.GP.tau(K))     # finish() multiplies by tau(K)
        return gemm_bound(c, mag, K)

    def weight_transpose_multi(c):
        if not is_x3(c.b):
            return wt_multi(c)
        out = []
        for i, ((w, _, s), (_, wt, _)) in enumerate(zip(c.b['jobs'], c.a['jobs'])):
            co, ci = w.shape[0], w.shape[-1]
            w3 = w.reshape(co, -1, ci)
            if s is not None:
                w3 = w3 * s.view(-1, 1, 1)     # one rounding in the tensors' dtype, as the kernel's product
            out.append(('jobs[%d]' % i, wt, w3.permute(2, 1, 0).reshape(wt.shape), None))
        return out

    class Audit(base):
        def _check(self, name, rec, b, a, ret, snaps):
            if name not in LA.GEMM_OPERANDS or not is_x3(b):
                return base._check(self, name, rec, b, a, ret, snaps)
            saved = LA.EXACTNESS_EXCEPTIONS
            LA.EXACTNESS_EXCEPTIONS = dict(saved)
            LA.EXACTNESS_EXCEPTIONS.update(((name, op), 'split-TF32 call: unrounded operands')
                                           for op in LA.GEMM_OPERANDS[name])
            try:
                return base._check(self, name, rec, b, a, ret, snaps)
            finally:
                LA.EXACTNESS_EXCEPTIONS = saved

    patch(LA, '_gemm_operand', operand)
    patch(LA, '_gemm_bound', bound)
    patch(LA, 'REF', dict(LA.REF, weight_transpose_multi=weight_transpose_multi))
    patch(LA, 'NETS', dict(LA.NETS, **NETS))
    patch(LA, 'Audit', Audit)


if __name__ == '__main__':
    install()
    sys.exit(LA.main())
