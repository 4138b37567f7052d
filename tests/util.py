"""Test helpers shared by the suites: TF32 rounding, sign-bit packing, NaN-guarded output buffers, the elementwise
comparison against fp64, the library's VLFB_DEBUG launch records and the GPU worker runner."""
import json
import os
import re
import subprocess
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)


def tf32_round(t):
    """cvt.rna.tf32.f32 (round to nearest, ties away) of the fp32 value of t, returned in t's dtype and shape."""
    i = t.float().contiguous().view(torch.int32)
    return ((i + 0x1000) & ~0x1FFF).view(torch.float32).to(t.dtype).view(t.shape)


def ulp_tf32(x):
    """One TF32 ulp (10 explicit mantissa bits) of |x|, elementwise; 0 at 0."""
    _, e = torch.frexp(x.abs())
    return torch.where(x == 0, torch.zeros_like(x), torch.ldexp(torch.ones_like(x), e - 11))


def pack_sign_bits(x):
    """bit e & 31 of word e >> 5 = x.flat[e] > 0 (vlfb_gemm_params_t.relu_bits_out / relu_mask_bits, vlfb_relu_bits)."""
    b = (x.reshape(-1, 32) > 0).to(torch.int64)
    v = (b << torch.arange(32, dtype=torch.int64, device=x.device)).sum(1)
    return torch.where(v >= 2 ** 31, v - 2 ** 32, v).to(torch.int32)


# ----------------------------------------------------------------------------------------------- guarded outputs
NAN_BITS = 0x7FC00000          # torch.full(..., nan) fills fp32 with this pattern; integer buffers get the same bits
BITS = {torch.float32: torch.int32, torch.bfloat16: torch.int16}


def nan_buffer(n, dev, dtype=torch.float32):
    """n elements of fill: NaN for fp32 / bf16, NAN_BITS for integer dtypes.  Outputs are placed inside such a buffer
    so that an element a kernel never writes, or writes out of range, is seen."""
    if dtype in BITS:
        return torch.full((n,), float('nan'), dtype=dtype, device=dev)
    return torch.full((n,), NAN_BITS, dtype=dtype, device=dev)


def guard_touched(buf, index):
    """Number of elements of the buffer `buf` outside the flat offsets `index` that no longer hold the fill bits."""
    bits = buf.reshape(-1)
    fill = nan_buffer(1, 'cpu', buf.dtype)
    if buf.dtype in BITS:
        bits, fill = bits.view(BITS[buf.dtype]), fill.view(BITS[buf.dtype])
    guard = torch.ones(bits.numel(), dtype=torch.bool, device=buf.device)
    guard[index.reshape(-1)] = False
    return int((bits[guard] != int(fill[0])).sum())


# ----------------------------------------------------------------------------------------------- comparison
def compare(got, ref, bound, tol=None, tol_rows=None):
    """got against its fp64 reference.  bound None: bit for bit (through an integer view for fp32 and bf16) and
    finite.  Otherwise every element finite and |got - ref| <= bound (an exact element counts as ratio 0), and, with
    `tol`, the global max|got - ref| / max|ref| < tol over the elements `tol_rows` selects (all by default).  Returns a
    dict: ok, nbad (elements outside the bound), nonfinite, worst_ratio |got - ref| / bound, worst_at (its index in
    ref's shape), rel_err."""
    shape = tuple(ref.shape)
    nonfinite = int((~torch.isfinite(got)).sum()) if got.dtype.is_floating_point else 0
    if bound is None:
        g, r = got.contiguous(), ref.to(got.dtype).reshape(got.shape).contiguous()
        if g.dtype in BITS:
            g, r = g.view(BITS[g.dtype]), r.view(BITS[g.dtype])
        bad = (g != r).reshape(-1)
        nbad = int(bad.sum())
        worst = int(bad.nonzero()[0]) if nbad else None
        worst_ratio, rel = (float('inf') if nbad else 0.0), 0.0
    else:
        d = got.double().reshape(shape)
        diff = (d - ref).abs()
        finite = torch.isfinite(d)
        ratio = torch.where(finite, diff / bound.clamp(min=1e-300), torch.full_like(diff, float('inf')))
        ratio = torch.where(diff == 0, torch.zeros_like(ratio), ratio)
        nbad = int((ratio > 1).sum())
        worst = int(ratio.reshape(-1).argmax()) if ratio.numel() else None
        worst_ratio = float(ratio.reshape(-1)[worst]) if worst is not None else 0.0
        sel = finite if tol_rows is None else finite & tol_rows
        if bool(sel.any()):
            rel = float(diff[sel].max() / (ref[sel].abs().max() + 1e-30))
        else:
            rel = 0.0 if bool(finite.all()) else float('inf')
    ok = nbad == 0 and nonfinite == 0 and (tol is None or rel < tol)
    at = [] if worst is None else [int(i) for i in np.unravel_index(worst, shape)]
    return dict(ok=ok, nbad=nbad, nonfinite=nonfinite, worst_ratio=worst_ratio, worst_at=at, rel_err=rel)


# ----------------------------------------------------------------------------------------------- launch records
def parse_record(line, kind='gemm_tc'):
    """One VLFB_DEBUG launch record 'vlfb <kind>: key=value ...' -> dict (None if the line is not one).  gemm_tc
    values are ints, with 'a,b' values as (a, b) tuples; gconv values stay strings."""
    m = re.search(r'vlfb %s:\s*(.*)$' % kind, line.strip())
    if not m:
        return None
    rec = {}
    for tok in m.group(1).split():
        if '=' not in tok:
            continue
        k, v = tok.split('=', 1)
        if kind == 'gemm_tc':
            v = tuple(int(x) for x in v.split(',')) if ',' in v else int(v)
        rec[k] = v
    return rec


def capture_fd2(fn):
    """Runs fn() with file descriptor 2 redirected to a temporary file (the library writes its VLFB_DEBUG records with
    fprintf(stderr)); returns (fn's result, the captured text)."""
    sys.stderr.flush()
    with tempfile.TemporaryFile() as tmp:
        saved = os.dup(2)
        os.dup2(tmp.fileno(), 2)
        try:
            out = fn()
        finally:
            sys.stderr.flush()
            os.dup2(saved, 2)
            os.close(saved)
        tmp.seek(0)
        text = tmp.read().decode('utf-8', 'replace')
    return out, text


# ----------------------------------------------------------------------------------------------- GPU workers
# Every environment override of the GEMM: a worker starts with none of them set except the ones it is given.
SWITCHES = ('VLFB_TMA', 'VLFB_IM2COL', 'VLFB_NO_PATCH', 'VLFB_NO_PAR', 'VLFB_BN', 'VLFB_STAGES', 'VLFB_LAG', 'VLFB_SK',
            'VLFB_DEBUG')
_WORKERS = {}


def run_worker(script, args, env=None, timeout=1800, tag=None, jsonl=True):
    """Runs tests/<script> with `args` in a fresh Python process from the repository root (the library reads its
    switches once per process), with every name of SWITCHES removed from the environment, then `env` applied and
    VLFB_DEBUG=1.  With `jsonl` the worker gets `--out FILE` and writes one JSON record per line there.  Returns
    (CompletedProcess, records or None).

    The outcome is kept for the session: a worker runs at most once per (script, args).  One that does not finish
    within `timeout` seconds is killed, and this call, and every later one for it, fails the calling test with the
    worker's last progress line (stdout lines starting with '[tag]'; tag defaults to the script's name)."""
    import pytest
    key = (script, tuple(args))
    if key not in _WORKERS:
        _WORKERS[key] = _start_worker(script, list(args), env or {}, timeout, tag or os.path.splitext(script)[0], jsonl)
    r = _WORKERS[key]
    if 'timeout' in r:
        pytest.fail('%s %s timed out after %d s; last progress line: %s' % (script, ' '.join(args), timeout,
                                                                            r['timeout']))
    return r['proc'], r['recs']


def _start_worker(script, args, env, timeout, tag, jsonl):
    e = dict((k, v) for k, v in os.environ.items() if k not in SWITCHES)
    e.update(env)
    e['VLFB_DEBUG'] = '1'
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.join(HERE, script)] + args
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, 'records.jsonl')
        try:
            proc = subprocess.run(cmd + (['--out', out] if jsonl else []), env=e, cwd=ROOT, capture_output=True,
                                  text=True, timeout=timeout)
        except subprocess.TimeoutExpired as ex:
            so = ex.stdout.decode() if isinstance(ex.stdout, bytes) else (ex.stdout or '')
            last = [l for l in so.splitlines() if l.startswith('[%s]' % tag)]
            return dict(timeout=last[-1] if last else '(none)')
        recs = None
        if jsonl:
            recs = []
            if os.path.exists(out):
                with open(out) as f:
                    recs = [json.loads(l) for l in f if l.strip()]
    return dict(proc=proc, recs=recs)


# ----------------------------------------------------------------------------------------------- layouts
def rel_err(a, b):
    """max|a-b| / max|b| -- the parity metric of SURVEY.md section 7."""
    a = a.detach().double().cpu()
    b = b.detach().double().cpu()
    return float((a - b).abs().max() / (b.abs().max() + 1e-30))


def to_cl(x):
    """NCTHW -> contiguous NDHWC."""
    return x.permute(0, 2, 3, 4, 1).contiguous()


def to_nc(x):
    """NDHWC -> contiguous NCTHW."""
    return x.permute(0, 4, 1, 2, 3).contiguous()


def w_to_cl(w):
    """(Co,Ci,kT,kH,kW) -> [Co,kT,kH,kW,Ci]."""
    return w.permute(0, 2, 3, 4, 1).contiguous()


def stem_pack(w):
    """(Co,3,kT,kH,kW<=8) -> [Co,kT,kH,8,4] zero padded (conv1 layout)."""
    co, ci, kt, kh, kw = w.shape
    out = torch.zeros((co, kt, kh, 8, 4), dtype=w.dtype)
    out[:, :, :, :kw, :ci] = w.permute(0, 2, 3, 4, 1)
    return out
