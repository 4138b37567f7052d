"""GPU diagnostic: error table of the tensor-core GEMM for every operand-major combination and
MN-major shared-memory layout mode (VLFB_MN_MODE).  Not a test; prints a table."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, 'video-long-term-feature-banks_b200', 'lib'))
sys.path.insert(0, os.path.join(ROOT, 'tests'))
from util import rel_err, tf32_round  # noqa: E402
from vlfb import kernels as K  # noqa: E402


def rnd(shape, seed):
    g = torch.Generator().manual_seed(seed)
    return tf32_round(torch.randn(shape, generator=g))


for backend in ('simt', 'tcgen05'):
    for mode in ((0, 1) if backend == 'tcgen05' else (0,)):
        os.environ['VLFB_MN_MODE'] = str(mode)
        K.set_gemm_backend(backend)
        for (B, M, N, Kd) in [(1, 128, 128, 64), (2, 256, 64, 32), (1, 128, 32, 8), (2, 392, 196, 128)]:
            for ta in (0, 1):
                for tb in (0, 1):
                    a = rnd((B, Kd, M) if ta else (B, M, Kd), 1)
                    b = rnd((B, N, Kd) if tb else (B, Kd, N), 2)
                    A = a.transpose(1, 2) if ta else a
                    Bm = b.transpose(1, 2) if tb else b
                    ref = torch.bmm(A.double(), Bm.double())
                    ad, bd = a.cuda(), b.cuda()
                    d = torch.full((B, M, N), float('nan'), device='cuda')
                    try:
                        K.matmul(ad.transpose(1, 2) if ta else ad, bd.transpose(1, 2) if tb else bd, d)
                        torch.cuda.synchronize()
                        e = rel_err(d, ref)
                    except Exception as ex:  # noqa
                        e = repr(ex)[:80]
                    print('%-8s mode=%d B=%d M=%d N=%d K=%d A=%s B=%s  err=%s' % (
                        backend, mode, B, M, N, Kd, 'MN' if ta else 'K ', 'K ' if tb else 'MN', e), flush=True)
