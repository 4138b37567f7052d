"""The weight-gradient GEMM (DENSE_MN x CONV_MN / STEM_MN / DENSE_MN, atomic epilogue) against fp64 at every production
geometry of R50-I3D-NL at 2 clips (tests/wgrad_cases.py) and at small ragged ones: K (positions) not a multiple of 64,
Co = 1, 32, 64 and 65, N tails, and stream-K / split-K schedules of each operand form.

These launches stage both operands by cp.async and publish each chunk by the completion of its copies
(cp.async.mbarrier.arrive), so the producers run ahead of the MMAs by the whole ring.  Each case is one conv_wgrad call whose result must lie within the elementwise bound
tau(K) of tests/gemm_paths.py, leave the NaN guard band around dw untouched and take the declared path.  The cases run in
a worker process (the library reads VLFB_DEBUG once, when it loads):

    VLFB_DEBUG=1 python tests/test_gpu_wgrad_pipeline.py --out FILE
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


def _case(name, seed, shape, co, ker, st=(1, 1, 1), pd=(0, 0, 0), dil=(1, 1, 1), opts=None, **expect):
    n, t, h, w, c = shape
    case = dict(name=name, op='conv_wgrad', seed=seed, opts=opts or {},
                geom=GP.G(n, t, h, w, c, co, tuple(ker), st=tuple(st), pd=tuple(pd), dil=tuple(dil)))
    run = dict(kinds=GP.describe(case)['kinds'], tma=(0, 0), cp=1)
    if c == 4:
        run['patch'] = 0
    run.update(expect)
    case['runs'] = {'default': run}
    return case


def cases():
    out = []
    for i, (label, shape, co, ker, st, pd, dil, _) in enumerate(WC.PRODUCTION):
        out.append(_case('prod ' + label, 500 + i, shape, co, ker, st, pd, dil))
    out += [
        # Co = 4 / 32 / 64 / 68 (M tails; the tensor-core wgrad needs Co % 4 == 0, 16-byte dY rows), positions not a
        # multiple of 64, N tails against the tile width
        _case('ragged M=4 3x3', 601, (1, 2, 6, 6, 32), 4, (1, 3, 3), pd=(0, 1, 1)),
        _case('ragged M=32 3x3 N tail', 602, (2, 3, 5, 7, 64), 32, (1, 3, 3), pd=(0, 1, 1)),
        _case('ragged M=64 3x1x1', 603, (1, 3, 10, 10, 32), 64, (3, 1, 1), pd=(1, 0, 0)),
        _case('ragged M=68 1x1', 604, (2, 2, 9, 9, 64), 68, (1, 1, 1)),
        _case('ragged M=68 3x3 N tail', 605, (1, 3, 7, 9, 32), 68, (1, 3, 3), pd=(0, 1, 1)),
        _case('ragged stem 5x7x7', 606, (1, 3, 20, 20, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3)),
        # stream-K (atomic, no fix-up) of each operand form
        _case('stream-K 3x3', 611, (2, 8, 14, 14, 128), 128, (1, 3, 3), pd=(0, 1, 1), opts=dict(stream_k=1), sk=1, fix=0),
        _case('stream-K 1x1', 612, (2, 16, 14, 14, 256), 128, (1, 1, 1), opts=dict(stream_k=1), sk=1, fix=0),
        _case('stream-K stem', 613, (1, 4, 36, 64, 4), 64, (5, 7, 7), st=(1, 2, 2), pd=(2, 3, 3), opts=dict(stream_k=1),
              sk=1, fix=0),
    ]
    return out


def check(K, c, dev):
    """One case -> its record (ok, errors, path, worst ratio to the bound, global relative error)."""
    import torch
    rec = dict(case=c['name'], errors=[])
    P = GP.prepare(c, dev)
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
    # the suite's global relative check, in the K range it was set for (beyond it the fp32 accumulation error of a
    # K-long sum grows with K; the elementwise bound above is the one that scales)
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
            print('[wgrad] %s' % c['name'], flush=True)
            try:
                rec = check(K, c, dev)
            except Exception as ex:                       # a failing call is a result of the case, not of the run
                rec = dict(case=c['name'], ok=False, paths=[], errors=['%s: %s' % (type(ex).__name__, ex)])
            f.write(json.dumps(rec) + '\n')
            f.flush()


@pytest.fixture(scope='module')
def records(tmp_path_factory):
    out = str(tmp_path_factory.mktemp('wgrad') / 'wgrad.jsonl')
    env = dict((k, v) for k, v in os.environ.items() if k not in GP.SWITCHES)
    env['VLFB_DEBUG'] = '1'
    cmd = [sys.executable] + (['-s'] if sys.flags.no_user_site else []) + [os.path.abspath(__file__), '--out', out]
    proc = subprocess.run(cmd, env=env, cwd=os.path.dirname(HERE), capture_output=True, text=True, timeout=TIMEOUT)
    assert proc.returncode == 0, 'worker exit %d\n%s\n%s' % (proc.returncode, proc.stdout[-3000:], proc.stderr[-3000:])
    with open(out) as f:
        return [json.loads(l) for l in f if l.strip()]


def test_wgrad_matches_fp64_and_declared_path(records):
    assert [r['case'] for r in records] == [c['name'] for c in cases()]
    bad = ['%s: %s' % (r['case'], '; '.join(r['errors'])) for r in records if not r['ok']]
    assert not bad, '\n  '.join(bad)


def test_wgrad_schedules_covered(records):
    """Every operand form (CONV_MN gathers, STEM_MN conv1, DENSE_MN pointwise) runs a split-K and a stream-K launch."""
    seen = set()
    for r in records:
        if r['ok'] and len(r['paths']) == 1:
            p = r['paths'][0]
            seen.add((p['kinds'][1], 'sk' if p['sk'] else ('split' if p['split'] > 1 else 'static')))
    missing = [(b, s) for b in (GP.OP_CONV_MN, GP.OP_STEM_MN, GP.OP_DENSE_MN) for s in ('sk', 'split') if (b, s) not in seen]
    assert not missing, 'not covered: %r' % missing


if __name__ == '__main__':
    main()
