"""Wide tiles of the tensor-core GEMM: a launch whose operands are both MN-major and whose M is at most 64 (every weight
gradient with Co <= 64) runs 64 x 2bn tiles, warpgroup w computing columns [w bn, (w + 1) bn) of the 64 rows, instead of
128 x bn tiles whose second warpgroup multiplies padding rows (csrc/gemm_tc.cu, Launch::wide).

Each case is one vlfb_gemm call checked against fp64 within tau(K) (tests/gemm_paths.py), with the NaN guard band around
its output intact and the declared path, `wide` included.  The cases cover every Co = 64 production geometry of
tests/wgrad_cases.py (and one Co = 128 that stays narrow), M = 4 / 32 / 60 / 64 against 68, N tails against bn and 2 bn,
forced tile widths, split-K and stream-K for each B operand kind, the row scale, the conv1 column mask, and a raw
DENSE_MN x DENSE_MN launch with a non-atomic ACCUM epilogue (every output element belongs to one warp: no reduction
across warpgroups).  The cases run in a worker process (the library reads VLFB_DEBUG once, when it loads):

    VLFB_DEBUG=1 python tests/test_gpu_wgrad_wide.py --out FILE
"""
import argparse
import json
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
if HERE not in sys.path:
    sys.path.insert(0, HERE)

import gemm_paths as GP  # noqa: E402
import wgrad_cases as WC  # noqa: E402

pytestmark = pytest.mark.gpu
TIMEOUT = 1800


def _case(name, seed, shape, co, ker, st=(1, 1, 1), pd=(0, 0, 0), dil=(1, 1, 1), opts=None, epi=None, col_mask=False,
          **expect):
    n, t, h, w, c = shape
    case = dict(name=name, op='conv_wgrad', seed=seed, opts=opts or {}, epi=epi or {}, col_mask=col_mask,
                geom=GP.G(n, t, h, w, c, co, tuple(ker), st=tuple(st), pd=tuple(pd), dil=tuple(dil)))
    run = dict(kinds=GP.describe(case)['kinds'], tma=(0, 0), cp=1, wide=1 if co <= 64 else 0)
    if c == 4:
        run['patch'] = 0
    run.update(expect)
    case['runs'] = {'default': run}
    return case


def cases():
    out = []
    co128 = 'res3_x_2b 1x3x3 128->128'
    for i, (label, shape, co, ker, st, pd, dil, _) in enumerate(WC.PRODUCTION):
        if co <= 64 or label == co128:
            out.append(_case('prod ' + label, 700 + i, shape, co, ker, st, pd, dil, wide=1 if co <= 64 else 0))
    rs = dict(row_scale=True)
    out += [
        # M against the 64-row wide tile (Co % 4 == 0: 16-byte dY rows)
        _case('M=4 3x3', 801, (1, 2, 6, 6, 32), 4, (1, 3, 3), pd=(0, 1, 1), epi=rs, wide=1),
        _case('M=32 3x3', 802, (2, 3, 5, 7, 64), 32, (1, 3, 3), pd=(0, 1, 1), wide=1),
        _case('M=60 3x1x1 N=32', 803, (1, 3, 8, 8, 32), 60, (3, 1, 1), pd=(1, 0, 0), epi=rs, wide=1),
        _case('M=64 1x1', 804, (2, 2, 9, 9, 64), 64, (1, 1, 1), wide=1),
        _case('M=68 3x3', 805, (1, 3, 7, 9, 32), 68, (1, 3, 3), pd=(0, 1, 1), wide=0),
        # N tails against bn and 2 bn, with the tile width forced
        _case('N=96 <= bn=128 1x1', 811, (2, 2, 8, 8, 96), 64, (1, 1, 1), opts=dict(tile_n=128), epi=rs, bn=128),
        _case('bn=64 < N=108 < 128 3x3', 812, (1, 3, 6, 6, 12), 48, (1, 3, 3), pd=(0, 1, 1), opts=dict(tile_n=64), bn=64),
        _case('N=144 = 2 x 64 + 16, bn=32 1x1', 813, (1, 4, 6, 6, 144), 64, (1, 1, 1), opts=dict(tile_n=32), epi=rs,
              bn=32),
        _case('N=144 = 128 + 16, bn=64 3x3', 814, (1, 3, 6, 6, 16), 64, (1, 3, 3), pd=(0, 1, 1), opts=dict(tile_n=64),
              bn=64),
        _case('N=224 bn=128 stem', 815, (1, 3, 20, 20, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3),
              opts=dict(tile_n=128), bn=128),
        # split-K (few wide tiles, long K) and stream-K (atomic, no fix-up) for each B operand kind
        _case('split-K CONV_MN', 821, (2, 8, 14, 14, 64), 64, (1, 3, 3), pd=(0, 1, 1), epi=rs, split='>1', sk=0),
        _case('split-K STEM_MN', 822, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), split='>1', sk=0),
        _case('split-K DENSE_MN', 823, (2, 8, 14, 14, 64), 64, (1, 1, 1), split='>1', sk=0),
        _case('stream-K CONV_MN', 831, (2, 8, 14, 14, 64), 64, (1, 3, 3), pd=(0, 1, 1), opts=dict(stream_k=1), sk=1, fix=0),
        _case('stream-K STEM_MN', 832, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3),
              opts=dict(stream_k=1), epi=rs, sk=1, fix=0),
        _case('stream-K DENSE_MN', 833, (2, 16, 28, 28, 64), 64, (1, 1, 1), opts=dict(stream_k=1), sk=1, fix=0),
        # conv1 with the optimiser's column mask (padding lanes px >= kW and the fourth channel zeroed) and a row scale
        _case('stem col_mask', 841, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), epi=rs, col_mask=True),
    ]
    # transposed x transposed matmul, M <= 64, plain stores with ACCUM (read-modify-write of D by exactly one warp)
    raw = dict(name='raw MNxMN M=48 accum', op='raw', seed=851, Z=2, M=48, N=200, K=300, a_mn=True, b_mn=True, gn=4,
               gm=2, epi=dict(accum=True, scale=True, bias=True, row_scale=True), opts={})
    raw['runs'] = {'default': dict(kinds=(GP.OP_DENSE_MN, GP.OP_DENSE_MN), tma=(0, 0), cp=1, wide=1, sk=0, split=1)}
    out.append(raw)
    return out


def _stem_mask(kH):
    """conv1's column mask: lane px * 4 + ch of a 32-lane filter row is real when px < kW (7) and ch < 3."""
    import torch
    m = torch.zeros(32)
    for px in range(7):
        m[px * 4:px * 4 + 3] = 1
    return m, m.repeat(kH)


def _run_col_mask(K, P, dev):
    """conv_wgrad with the 32-lane col_mask the optimiser passes for conv1 (GP.run_case passes no column scale)."""
    import torch
    c = P.case
    g = c['geom']
    buf = torch.full((P.layout['size'],), float('nan'), device=dev)
    flat = buf.view(-1)
    flat[P.index.reshape(-1)] = P.epi['prev'].reshape(-1).float()
    Z, M, N = P.ref.shape
    out = flat[GP.GUARD:GP.GUARD + Z * M * N]
    m32, _ = _stem_mask(g['ker'][1])
    rs = P.epi['rs'].float() if 'rs' in P.epi else None
    geo = K.conv_geom((g['N'], g['T'], g['H'], g['W'], g['C']), g['Co'], g['ker'], g['st'], g['pd'], g['dil'])
    x = GP._stem_input(K, P, dev)
    dw = out.view((g['Co'],) + tuple(g['ker'][:2]) + (8, 4))
    GP._opts(K, c)
    try:
        K.conv_wgrad(GP._to_cl(P.dy).to(dev), x, dw, geo, row_scale=rs, col_mask=m32.to(dev))
        torch.cuda.synchronize()
    finally:
        GP._opts(K, {'opts': {}})
    return buf, None


def check(K, c, dev):
    """One case -> its record (ok, errors, path, worst ratio to the bound, global relative error)."""
    import torch
    rec = dict(case=c['name'], errors=[])
    P = GP.prepare(c, dev)
    if c.get('col_mask'):
        _, full = _stem_mask(c['geom']['ker'][1])
        P.epi['cs'] = full.double().to(dev)
        P.ref, P.bound = GP.finish(P.acc, P.mag, P.epi, P.K)
        (buf, _), text = GP.capture_fd2(lambda: _run_col_mask(K, P, dev))
    else:
        (buf, _), text = GP.capture_fd2(lambda: GP.run_case(K, P, dev))
    paths = [r for r in (GP.parse_record(l) for l in text.splitlines()) if r is not None]
    rec['paths'] = [dict((k, list(v) if isinstance(v, tuple) else v) for k, v in r.items()) for r in paths]
    if len(paths) != 1:
        rec['errors'].append('expected one tensor-core launch record, got %d' % len(paths))
    else:
        want = GP.describe(c)
        for k in ('M', 'N', 'K'):
            if paths[0][k] != want[k]:
                rec['errors'].append('record %s=%d, case describes %d' % (k, paths[0][k], want[k]))
        bad = GP.matches(paths[0], c['runs']['default'])
        if bad:
            rec['errors'].append('path: ' + ', '.join(bad))
    d = buf.view(-1)[P.index.reshape(-1)].view(P.ref.shape)
    cmp = GP.compare(d, P.ref, P.bound)
    rec.update(worst_ratio=cmp['worst_ratio'], rel_err=cmp['rel_err'], K=P.K)
    if not cmp['ok']:
        rec['errors'].append('values: %d elements outside tau(K), %d not finite, worst %.3g x bound at %s' % (
            cmp['nbad'], cmp['nonfinite'], cmp['worst_ratio'], cmp['worst_at']))
    if P.K <= GP.KMAX and not cmp['rel_err'] < 2e-5:
        rec['errors'].append('global rel_err %.3g >= 2e-5' % cmp['rel_err'])
    touched = GP.guard_intact(buf, P.index)
    if touched:
        rec['errors'].append('%d guard elements overwritten' % touched)
    rec['ok'] = not rec['errors']
    del P, buf
    torch.cuda.empty_cache()
    return rec


def main(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split('\n')[0])
    ap.add_argument('--out', required=True)
    args = ap.parse_args(argv)
    if os.environ.get('VLFB_DEBUG') != '1':
        raise SystemExit('the path records need VLFB_DEBUG=1')
    import torch
    from vlfb import kernels as K
    dev = torch.device('cuda')
    K.set_gemm_backend('tcgen05')
    with open(args.out, 'w') as f:
        for c in cases():
            print('[wide] %s' % c['name'], flush=True)
            try:
                rec = check(K, c, dev)
            except Exception as ex:                       # a failing call is a result of the case, not of the run
                rec = dict(case=c['name'], ok=False, paths=[], errors=['%s: %s' % (type(ex).__name__, ex)])
            f.write(json.dumps(rec) + '\n')
            f.flush()


@pytest.fixture(scope='module')
def records(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('wide') / 'wide.jsonl')
    env = dict((k, v) for k, v in os.environ.items() if k not in GP.SWITCHES)
    env['VLFB_DEBUG'] = '1'
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), '--out', out]
    proc = subprocess.run(cmd, env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=TIMEOUT)
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    with open(out) as f:
        return [json.loads(l) for l in f if l.strip()]


def test_wide_matches_fp64_and_declared_path(records):
    assert [r['case'] for r in records] == [c['name'] for c in cases()]
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in records if not r['ok']]
    assert not bad, '\n  '.join(bad)


def test_wide_paths_covered(records):
    """Wide launches run every tile width, a split-K and a stream-K schedule of every B operand kind, and N tails."""
    seen = set()
    for r in records:
        if r['ok'] and len(r['paths']) == 1 and r['paths'][0].get('wide') == 1:
            p = r['paths'][0]
            seen.add(('bn', p['bn']))
            seen.add((p['kinds'][1], 'sk' if p['sk'] else ('split' if p['split'] > 1 else 'static')))
            if p['N'] <= p['bn']:
                seen.add('N <= bn')
            elif p['N'] < 2 * p['bn']:
                seen.add('bn < N < 2bn')
            elif p['N'] % (2 * p['bn']) == 16:
                seen.add('N = 2bn q + 16')
    want = [('bn', 32), ('bn', 64), ('bn', 128), 'N <= bn', 'bn < N < 2bn', 'N = 2bn q + 16']
    want += [(b, s) for b in (GP.OP_CONV_MN, GP.OP_STEM_MN, GP.OP_DENSE_MN) for s in ('sk', 'split')]
    missing = [w for w in want if w not in seen]
    assert not missing, 'not covered: %r' % missing


if __name__ == '__main__':
    main()
