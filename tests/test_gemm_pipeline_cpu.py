"""The wgmma pipeline of the tensor-core GEMM, checked on the compiler output (no GPU needed).

gemm_tc.cu is compiled for sm_90a with the build's nvcc flags plus `-Xptxas -v`, and `cuobjdump -sass` lists what ptxas
made of every gemm_tc_kernel instantiation.  ptxas silently falls back to running each wgmma to completion before the
next one when it cannot prove the asynchronous pipeline safe (it then reports "wgmma.mma_async instructions are
serialized", C7510-C7519, and injects warpgroup waits, C7517).  Nothing fails at run time; the kernel only gets slower.
These tests pin the pipeline down:
  - no "serialized" report and no injected wait;
  - the 4 HGMMA of a 32-k chunk are issued back to back: no `WARPGROUP.DEPBAR.LE gsb0, 0x0` (full drain) between them;
  - every K loop waits with `DEPBAR.LE gsb0, 0x1` (the previous chunk's MMAs stay in flight);
  - MN-major B with a K-major A (transposed matmul B operands): no full drain inside the K loop at all; MN-major A
    (wgrad, transposed matmul A operands): one drain per chunk, for the single A image;
  - no register spills, except in two stream-K fix-up builds at the 168-register cap, which may not grow;
  - exactly the expected instantiations are built: TMA-only builds (CP = false) for K-major operand pairs only.
"""
import os
import re
import shutil
import subprocess
import tempfile

import pytest

import __graft_entry__ as G

SRC = os.path.join(G.CSRC, 'gemm_tc.cu')
MN_KINDS = {1, 4, 6}                 # VLFB_OP_DENSE_MN, VLFB_OP_CONV_MN, VLFB_OP_STEM_MN (include/vlfb.h)
# (A kind, B kind, MASK, CP, FIX) -> spill-store bytes allowed
# The two MASK builds spilled before the pipeline was restored.
SPILL_ALLOWED = {(0, 0, 1, 0, 1): 24, (3, 0, 1, 0, 1): 12}
MMA_PER_CHUNK = 4                    # 32 fp32 of K per chunk / wgmma k8
# (A kind, B kind, MASK) of every launch gemm_tc() dispatches (kinds: include/vlfb.h)
DISPATCHED = [(2, 0, 0), (5, 0, 0), (3, 0, 0), (1, 4, 0), (1, 6, 0), (0, 0, 0), (0, 1, 0), (1, 0, 0), (1, 1, 0),
              (3, 0, 1), (0, 0, 1)]


def expected_builds():
    """(A kind, B kind, MASK, CP, FIX) of every gemm_tc_kernel instantiation.  A pair with an MN-major operand is staged
    (partly) by cp.async, so it has only CP = true builds: FIX = 0, and FIX = 1 for the MN x MN pairs without a mask
    (the cp.async fix-up of deterministic launches).  A K-major pair has the cp.async build and both TMA-only builds."""
    out = set()
    for ak, bk, mask in DISPATCHED:
        if ak in MN_KINDS or bk in MN_KINDS:
            out.add((ak, bk, mask, 1, 0))
            if ak in MN_KINDS and bk in MN_KINDS and not mask:
                out.add((ak, bk, mask, 1, 1))
        else:
            out.update({(ak, bk, mask, 1, 0), (ak, bk, mask, 0, 0), (ak, bk, mask, 0, 1)})
    return out

NAME_RE = re.compile(r'_ZN4vlfb2tc14gemm_tc_kernelILi(\d+)ELi(\d+)ELb(\d)ELb(\d)ELb(\d)EEEv\w*')
INSN_RE = re.compile(r'/\*([0-9a-f]{4,})\*/\s+([^;]*);')
BRA_RE = re.compile(r'\bBRA(?:\.\S+)?\s+`?\(?(0x[0-9a-f]+)')


def _tool(name):
    nvcc = os.environ.get('NVCC', 'nvcc')
    path = shutil.which(nvcc)
    if path is None:
        return None
    return path if name == 'nvcc' else shutil.which(os.path.join(os.path.dirname(path), name))


def _key(mangled):
    m = NAME_RE.match(mangled)
    return tuple(int(x) for x in m.groups()) if m else None


def _fmt(key):
    return 'kinds=%d,%d mask=%d cp=%d fix=%d' % key


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
    return parse(log, sass)


def parse(log, sass):
    """ptxas -v log + cuobjdump -sass text -> per instantiation key: registers / spills, ptxas diagnostics, SASS."""
    # ptxas -v: per entry function its spills and registers; every diagnostic names the function it is about
    info, diags = {}, {}
    cur = None
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
    # SASS: per function the instruction list in address order
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
    assert funcs, 'no gemm_tc_kernel instantiation in the SASS'
    return dict(info=info, diags=diags, funcs=funcs)


def _chunks(body):
    """Indices (into body) of the HGMMA of each K chunk: consecutive groups of MMA_PER_CHUNK in program order."""
    h = [i for i, (_, ins) in enumerate(body) if ins.startswith('HGMMA')]
    return [h[j:j + MMA_PER_CHUNK] for j in range(0, len(h), MMA_PER_CHUNK)], len(h)


def _is_drain(ins):
    return ins.startswith('WARPGROUP.DEPBAR.LE') and ins.endswith('0x0')


def _k_loop(body, chunk):
    """[first, last] instruction index of the innermost loop (backward branch) around one chunk's HGMMA."""
    lo_addr, hi_addr = body[chunk[0]][0], body[chunk[-1]][0]
    best = None
    for i, (addr, ins) in enumerate(body):
        m = BRA_RE.search(ins)
        if not m:
            continue
        tgt = int(m.group(1), 16)
        if tgt <= lo_addr and addr >= hi_addr and (best is None or addr - tgt < best[1] - best[0]):
            best = (tgt, addr)
    assert best is not None, 'no loop around the HGMMA at %#x' % lo_addr
    return [i for i, (addr, _) in enumerate(body) if best[0] <= addr <= best[1]]


def test_every_instantiation_is_reported(compiled):
    assert set(compiled['funcs']) == set(compiled['info']), 'ptxas -v and cuobjdump list different kernels'
    for key, body in compiled['funcs'].items():
        chunks, n = _chunks(body)
        assert n and n % MMA_PER_CHUNK == 0, '%s: %d HGMMA' % (_fmt(key), n)


def test_instantiations_are_exactly_the_dispatched_builds(compiled):
    want = expected_builds()
    assert len(want) == 26
    got = set(compiled['funcs'])
    assert got == want, 'unexpected: %s; missing: %s' % (sorted(map(_fmt, got - want)), sorted(map(_fmt, want - got)))


def test_no_serialized_wgmma(compiled):
    bad = ['%s: %s' % (_fmt(k), d) for k, ds in sorted(compiled['diags'].items()) for d in ds
           if 'serialized' in d or 'C7517' in d or re.search(r'\(C751\d\)', d)]
    assert not bad, '\n'.join(bad)


def test_no_spills(compiled):
    bad = []
    for key, rec in sorted(compiled['info'].items()):
        allowed = SPILL_ALLOWED.get(key, 0)
        if rec.get('spill_st', 0) > allowed or rec.get('spill_ld', 0) > allowed:
            bad.append('%s: %d B spill stores, %d B spill loads (allowed %d)' % (_fmt(key), rec['spill_st'], rec['spill_ld'], allowed))
    assert not bad, '\n'.join(bad)


def test_chunk_mmas_issue_back_to_back(compiled):
    bad = []
    for key, body in sorted(compiled['funcs'].items()):
        chunks, _ = _chunks(body)
        for c in chunks:
            drains = [body[i][0] for i in range(c[0], c[-1]) if _is_drain(body[i][1])]
            if drains:
                bad.append('%s: full drain at %s inside the chunk %#x..%#x' %
                           (_fmt(key), ', '.join('%#x' % a for a in drains), body[c[0]][0], body[c[-1]][0]))
    assert not bad, '\n'.join(bad[:40])


def test_k_loop_keeps_one_chunk_in_flight(compiled):
    """Every K loop (one per tile width) waits for the previous chunk with DEPBAR.LE gsb0, 0x1."""
    bad = []
    for key, body in sorted(compiled['funcs'].items()):
        chunks, _ = _chunks(body)
        for c in chunks:
            if not any(body[i][1] == 'WARPGROUP.DEPBAR.LE gsb0, 0x1' for i in _k_loop(body, c)):
                bad.append('%s: no DEPBAR.LE gsb0, 0x1 in the K loop of the chunk at %#x' % (_fmt(key), body[c[0]][0]))
    assert not bad, '\n'.join(bad[:40])


def test_mn_major_k_loop_drains(compiled):
    """An MN-major B is rewritten into one of two K-major images while the previous chunk's MMAs read the other: with
    a K-major A its K loop never drains.  An MN-major A has one K-major image, so its K loop drains exactly once per
    chunk, before the rewrite (the A operand from registers, which would remove that drain, is not used: DESIGN.md 4.1)."""
    bad = []
    for key, body in sorted(compiled['funcs'].items()):
        if key[0] not in MN_KINDS and key[1] not in MN_KINDS:
            continue
        allowed = 1 if key[0] in MN_KINDS else 0
        chunks, _ = _chunks(body)
        for c in chunks:
            drains = [body[i][0] for i in _k_loop(body, c) if _is_drain(body[i][1])]
            if len(drains) > allowed:
                bad.append('%s: %d full drains in the K loop at %s (allowed %d)' %
                           (_fmt(key), len(drains), ', '.join('%#x' % a for a in drains), allowed))
    assert not bad, '\n'.join(bad[:40])
