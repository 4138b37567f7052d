"""The launch audit (tests/launch_audit.py) checked without a GPU: the tiny AVA FBO-NL train step runs on the CPU
stand-in (tests/fake_kernels.py in fp32, TF32 roundings emulated) through the interposer, with the case tables' references as
the oracle and the TF32-exactness check on.  It must pass; every planted fault must be flagged at exactly the wrapper
it is planted in, with a message naming the net step."""
import pytest
import torch

import launch_audit as LA


@pytest.fixture
def fake():
    import fake_kernels
    from vlfb import executor, workspace
    executor.set_backend(fake_kernels, 'cpu', torch.float32)      # the kernels' dtype: the fp32 bounds are meaningful
    fake_kernels.EMULATE_TF32 = True
    workspace.ResetWorkspace()
    yield fake_kernels
    fake_kernels.EMULATE_TF32 = False
    workspace.ResetWorkspace()
    fake_kernels.uninstall()


def _audit(fake, runs=None):
    audit = LA.Audit(fake, 'fake_tf32')
    missing = LA.run_net(audit, 'ava_train', runs=runs)
    return audit, missing


def test_tiny_ava_train_step_passes_the_audit(fake):
    audit, missing = _audit(fake)
    print('\n' + LA.report(audit))
    assert not missing, missing
    bad = audit.failures()
    assert not bad, '\n'.join(e for r in bad[:10] for e in r['errors'])
    assert {r['run'] for r in audit.records} == {0, 1, 2}          # run 0: feeding the parameters and inputs
    # every wrapper the executor reached has a reference (a missing one is an error, not a skip)
    assert set(audit.calls) <= set(LA.REF)
    for r in audit.records:
        assert r['outputs'], r['wrapper']


def test_fake_matmul_declines_rounding_of_split_products(fake):
    """kernels.matmul returns False for tf32_optional products it splits over K (few tiles, K >= 1024); the stand-in
    must too, and an accumulated product with tf32_out is stored rounded."""
    a = torch.randn(1, 8, 2048, dtype=torch.float64)
    b = torch.randn(1, 2048, 16, dtype=torch.float64)
    d = torch.zeros(1, 8, 16, dtype=torch.float64)
    assert fake.matmul(a, b, d, tf32_out=True, tf32_optional=True) is False
    assert fake.matmul(a, b, d, tf32_out=True) is True
    assert fake.matmul(a[:, :, :64], b[:, :64], d, tf32_out=True, tf32_optional=True) is True
    d0 = torch.randn(1, 8, 16, dtype=torch.float64)
    d = d0.clone()
    fake.matmul(a[:, :, :64], b[:, :64], d, accumulate=True, tf32_out=True)
    assert LA.not_tf32_exact(d) == 0
    assert torch.allclose(d, d0 + torch.bmm(a[:, :, :64], b[:, :64]), rtol=1e-3, atol=1e-3)


def _flagged(audit):
    """The wrappers with a failing call; every failure message must name its net step (the executor's K.LABEL)."""
    for r in audit.failures():
        assert r['label'], r['errors'][:2]
        for e in r['errors']:
            assert "ava_train run %d step %r %s" % (r['run'], r['label'], r['wrapper']) in e, e
    return {r['wrapper'] for r in audit.failures()}


def _plant(monkeypatch, fake, name, f):
    monkeypatch.setattr(fake, name, f)


def test_audit_flags_a_dgrad_that_ignores_accumulate(fake, monkeypatch):
    orig = fake.conv_dgrad

    def bad(dy, wt, dx, g, accumulate=False, **kw):
        return orig(dy, wt, dx, g, accumulate=False, **kw)
    _plant(monkeypatch, fake, 'conv_dgrad', bad)
    audit, _ = _audit(fake, runs=1)
    assert _flagged(audit) == {'conv_dgrad'}


def test_audit_flags_a_conv_fwd_that_drops_the_last_channels_bias(fake, monkeypatch):
    orig = fake.conv_fwd

    def bad(x, w, y, g, scale=None, bias=None, **kw):
        if bias is not None:
            bias = bias.clone()
            bias[-1] = 0
        return orig(x, w, y, g, scale=scale, bias=bias, **kw)
    _plant(monkeypatch, fake, 'conv_fwd', bad)
    audit, _ = _audit(fake, runs=1)
    assert _flagged(audit) == {'conv_fwd'}


def test_audit_flags_a_relu_mask_tested_with_ge(fake, monkeypatch):
    def bad(dy, y, dx):
        dx.copy_(fake._q(dy * (y >= 0)))
    _plant(monkeypatch, fake, 'relu_bwd_tf32', bad)
    audit, _ = _audit(fake, runs=1)
    assert _flagged(audit) == {'relu_bwd_tf32'}


def test_audit_flags_a_round_tf32_that_truncates(fake, monkeypatch):
    def bad(x, y):
        y.copy_(LA.tf32_trunc(x))
    _plant(monkeypatch, fake, 'round_tf32', bad)
    audit, _ = _audit(fake, runs=1)
    assert _flagged(audit) == {'round_tf32'}


def test_audit_flags_copy2d_writing_past_cols(fake, monkeypatch):
    orig = fake.copy2d

    def bad(src, lds, dst, ldd, rows, cols, accumulate=False, src_off=0, dst_off=0):
        orig(src, lds, dst, ldd, rows, cols, accumulate, src_off, dst_off)
        flat = torch.as_strided(dst, (dst.untyped_storage().nbytes() // dst.element_size(),), (1,), 0)
        i = dst.storage_offset() + dst_off + cols
        if i < flat.numel():          # the lowest mantissa bit of the element after row 0: the smallest change there is
            flat[i:i + 1].view(torch.int32).bitwise_xor_(1)
    _plant(monkeypatch, fake, 'copy2d', bad)
    audit, _ = _audit(fake, runs=1)
    assert _flagged(audit) == {'copy2d'}


def test_audit_flags_an_executor_rounding_lapse_as_an_inexact_gemm_operand(fake, monkeypatch):
    """Ctx.rounded hands a GEMM its operand unrounded: only the exactness check can see it (the stand-in computes with
    whatever it is given), and it must name the GEMM that read it."""
    from vlfb import executor as X

    def lapse(self, name):
        if self.ws.params.has(name):
            return self.ws.params.tf32(name)
        return self.ws.blobs[name]
    monkeypatch.setattr(X.Ctx, 'rounded', lapse)
    audit, _ = _audit(fake, runs=1)
    flagged = _flagged(audit)
    assert flagged and flagged <= set(LA.GEMM_WRAPPERS), flagged
    errs = [e for r in audit.failures() for e in r['errors']]
    assert all('not TF32-exact' in e for e in errs), errs[:5]
