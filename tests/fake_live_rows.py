"""TEST-ONLY: the `live_rows` argument of the kernels a B200.ROI_CAPACITY net passes it to (include/vlfb_live.h,
vlfb_fbo_cfg_t.live_rows), on top of the torch-CPU stand-in of tests/fake_kernels.py.  Each wrapper runs the stand-in
over rows [0, live) only -- what a launch over the live rows alone computes -- and writes zeros to the padded rows of
its outputs, as the CUDA kernels do.  install(monkeypatch) routes the stand-in's functions through them."""
import fake_kernels as F

FBO_ACTS = ('theta', 'prob', 's', 't', 'xhat', 'ln_mean', 'ln_std', 'out', 'a_out')


def _rows(live_rows, rows):
    return rows if live_rows is None else int(live_rows.view(-1)[0])


def roi_align_fwd(feat, rois, out, spatial_scale, sampling_ratio=0, live_rows=None):
    n = _rows(live_rows, rois.shape[0])
    _orig['roi_align_fwd'](feat, rois[:n], out[:n], spatial_scale, sampling_ratio)
    out[n:].zero_()


def roi_align_bwd(dout, rois, dfeat, spatial_scale, sampling_ratio=0, live_rows=None):
    n = _rows(live_rows, rois.shape[0])
    _orig['roi_align_bwd'](dout[:n], rois[:n], dfeat, spatial_scale, sampling_ratio)


def fbo_bank_scan(bank, q, out, scale, prob=None, tf32_out=False, live_rows=None):
    n = _rows(live_rows, bank.shape[0])
    _orig['fbo_bank_scan'](bank[:n], q[:n], out[:n], scale, prob=None if prob is None else prob[:n], tf32_out=tf32_out)
    out[n:].zero_()
    if prob is not None:
        prob[n:].zero_()


def _live_cfg(cfgd, rows):
    n = _rows(cfgd.get('live_rows'), rows)
    cfg = dict((k, v) for k, v in cfgd.items() if k != 'live_rows')
    cfg['R'] = n
    return cfg, n


def fbo_nl_fwd(cfgd, layers, a0, bp):
    cfg, n = _live_cfg(cfgd, a0.shape[0])
    _orig['fbo_nl_fwd'](cfg, [dict(ld, **dict((k, ld[k][:n]) for k in FBO_ACTS)) for ld in layers], a0[:n], bp[:n])
    for ld in layers:
        for k in FBO_ACTS:
            ld[k][n:].zero_()


def fbo_nl_bwd(cfgd, layers, a0, bp, da_last, da0, dbp):
    cfg, n = _live_cfg(cfgd, a0.shape[0])
    _orig['fbo_nl_bwd'](cfg, layers, a0[:n], bp[:n], da_last[:n], da0[:n], dbp[:n])
    da0[n:].zero_()
    dbp[n:].zero_()


_WRAPPED = ('roi_align_fwd', 'roi_align_bwd', 'fbo_bank_scan', 'fbo_nl_fwd', 'fbo_nl_bwd')
_orig = dict((name, getattr(F, name)) for name in _WRAPPED)


def install(monkeypatch):
    for name in _WRAPPED:
        monkeypatch.setattr(F, name, globals()[name])
