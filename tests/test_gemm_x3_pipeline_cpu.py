"""The wgmma pipeline of the split-TF32 GEMM (gemm_tc3_kernel, vlfb_gemm_params_t.precision = VLFB_PREC_X3), checked on
the compiler output (no GPU needed), as tests/test_gemm_pipeline_cpu.py checks gemm_tc_kernel.

A split chunk issues 3 MMAs per k8 step (A_hi B_lo, A_lo B_hi, A_hi B_hi), 12 per 32-k chunk.  For every instantiation:
  - no "serialized" report (C7510-C7519) and no injected warpgroup wait (C7517);
  - no register spills, except one word in each of the two TMA-only stream-K fix-up builds with a ReLU mask, at the
    168-register cap (their TF32 forms are the builds tests/test_gemm_pipeline_cpu.py allows 24 and 12 bytes), which may
    not grow;
  - the 12 HGMMA of a chunk are issued back to back (no `WARPGROUP.DEPBAR.LE gsb0, 0x0` between them);
  - every K loop waits with `DEPBAR.LE gsb0, 0x1`, so the previous chunk's MMAs stay in flight while the consumers
    build the next chunk's lo images;
  - the instantiation set is exactly that of gemm_tc_kernel: every launch path has its split form.
"""
import os
import re
import subprocess
import tempfile

import pytest

import __graft_entry__ as G
from test_gemm_pipeline_cpu import INSN_RE, _is_drain, _k_loop, _tool, expected_builds

SRC = os.path.join(G.CSRC, 'gemm_tc.cu')
MMA_PER_CHUNK = 12                   # 32 fp32 of K per chunk / wgmma k8, three products per step
SPILL_ALLOWED = {(0, 0, 1, 0, 1): 4, (3, 0, 1, 0, 1): 4}  # (A kind, B kind, MASK, CP, FIX) -> spill bytes allowed
NAME_RE = re.compile(r'_ZN4vlfb2tc15gemm_tc3_kernelILi(\d+)ELi(\d+)ELb(\d)ELb(\d)ELb(\d)EEEv\w*')


def _key(mangled):
    m = NAME_RE.match(mangled)
    return tuple(int(x) for x in m.groups()) if m else None


def _fmt(key):
    return 'x3 kinds=%d,%d mask=%d cp=%d fix=%d' % key


@pytest.fixture(scope='module')
def compiled():
    nvcc, cuobjdump = _tool('nvcc'), _tool('cuobjdump')
    if nvcc is None or cuobjdump is None:
        pytest.skip('nvcc / cuobjdump not found')
    with tempfile.TemporaryDirectory() as tmp:
        obj = os.path.join(tmp, 'gemm_tc.o')
        r = subprocess.run([nvcc] + G.NVCC_FLAGS + ['-Xptxas', '-v', '-c', SRC, '-o', obj],
                           capture_output=True, text=True, timeout=1800)
        assert r.returncode == 0, r.stderr[-4000:]
        log = r.stdout + r.stderr
        sass = subprocess.run([cuobjdump, '-sass', obj], capture_output=True, text=True, check=True, timeout=600).stdout
    info, diags, cur = {}, {}, None
    for line in log.splitlines():
        m = re.search(r"Function properties for (\S+)", line) or re.search(r"Compiling entry function '(\S+)'", line)
        if m:
            cur = _key(m.group(1))
            if cur is not None:
                info.setdefault(cur, {})
            continue
        m = re.search(r"function '(\S+)'", line)
        if m and _key(m.group(1)) is not None:
            diags.setdefault(_key(m.group(1)), []).append(line.strip())
            continue
        if cur is None:
            continue
        m = re.search(r'(\d+) bytes spill stores, (\d+) bytes spill loads', line)
        if m:
            info[cur]['spill_st'], info[cur]['spill_ld'] = int(m.group(1)), int(m.group(2))
        m = re.search(r'Used (\d+) registers', line)
        if m:
            info[cur]['regs'] = int(m.group(1))
    funcs, body = {}, None
    for line in sass.splitlines():
        m = re.search(r'Function : (\S+)', line)
        if m:
            k = _key(m.group(1))
            body = funcs.setdefault(k, []) if k is not None else None
            continue
        if body is not None:
            m = INSN_RE.search(line)
            if m:
                body.append((int(m.group(1), 16), ' '.join(m.group(2).split())))
    assert funcs, 'no gemm_tc3_kernel instantiation in the SASS'
    return dict(info=info, diags=diags, funcs=funcs)


def _chunks(body):
    h = [i for i, (_, ins) in enumerate(body) if ins.startswith('HGMMA')]
    return [h[j:j + MMA_PER_CHUNK] for j in range(0, len(h), MMA_PER_CHUNK)], len(h)


def test_split_instantiations_are_exactly_the_dispatched_builds(compiled):
    assert set(compiled['funcs']) == set(compiled['info']), 'ptxas -v and cuobjdump list different kernels'
    got, want = set(compiled['funcs']), expected_builds()
    assert got == want, 'unexpected: %s; missing: %s' % (sorted(map(_fmt, got - want)), sorted(map(_fmt, want - got)))
    for key, body in compiled['funcs'].items():
        _, n = _chunks(body)
        assert n and n % MMA_PER_CHUNK == 0, '%s: %d HGMMA' % (_fmt(key), n)


def test_split_no_serialized_wgmma(compiled):
    bad = ['%s: %s' % (_fmt(k), d) for k, ds in sorted(compiled['diags'].items()) for d in ds
           if 'serialized' in d or 'C7517' in d or re.search(r'\(C751\d\)', d)]
    assert not bad, '\n'.join(bad)


def test_split_no_spills(compiled):
    bad = ['%s: %d B spill stores, %d B spill loads' % (_fmt(k), r.get('spill_st', 0), r.get('spill_ld', 0))
           for k, r in sorted(compiled['info'].items())
           if max(r.get('spill_st', 0), r.get('spill_ld', 0)) > SPILL_ALLOWED.get(k, 0)]
    assert not bad, '\n'.join(bad)


def test_split_chunk_mmas_issue_back_to_back(compiled):
    bad = []
    for key, body in sorted(compiled['funcs'].items()):
        chunks, _ = _chunks(body)
        for c in chunks:
            drains = [body[i][0] for i in range(c[0], c[-1]) if _is_drain(body[i][1])]
            if drains:
                bad.append('%s: full drain at %s inside the chunk %#x..%#x' %
                           (_fmt(key), ', '.join('%#x' % a for a in drains), body[c[0]][0], body[c[-1]][0]))
    assert not bad, '\n'.join(bad[:40])


def test_split_k_loop_keeps_one_chunk_in_flight(compiled):
    bad = []
    for key, body in sorted(compiled['funcs'].items()):
        chunks, _ = _chunks(body)
        for c in chunks:
            if not any(body[i][1] == 'WARPGROUP.DEPBAR.LE gsb0, 0x1' for i in _k_loop(body, c)):
                bad.append('%s: no DEPBAR.LE gsb0, 0x1 in the K loop of the chunk at %#x' % (_fmt(key), body[c[0]][0]))
    assert not bad, '\n'.join(bad[:40])
