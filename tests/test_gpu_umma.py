"""Known-answer test of the tensor-core plumbing (csrc/wgmma.cuh): one CTA of two warpgroups computes D[128, N] = A[128, K] . B[N, K]^T
with wgmma.mma_async (TF32 inputs, FP32 accumulators in registers), A from per-thread register fragments and B from K-major,
unswizzled shared memory.  The Leung-Malik contraction (csrc/lm_texture.cu) uses exactly these operand layouts and descriptor
encodings, at its two widths N = 48 and N = 80."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tf32(x):
    bits = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


@pytest.mark.parametrize('N,K', [(80, 40), (48, 40), (80, 8), (48, 64)])
def test_wgmma_tf32_gemm_known_answer(N, K):
    from pyimsegm_b200 import _lib
    torch = _lib.require_cuda()
    lib = _lib.lib()
    rng = np.random.RandomState(7 * N + K)
    A = _tf32(rng.standard_normal((128, K)).astype(np.float32))
    B = _tf32(rng.standard_normal((N, K)).astype(np.float32))
    want = A.astype(np.float64) @ B.astype(np.float64).T
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    dD = torch.zeros((128, N), dtype=torch.float32, device='cuda')
    _lib.check(lib.isb_wgmma_selftest(_lib.ptr(dA), _lib.ptr(dB), N, K, 2, _lib.ptr(dD), _lib.stream_ptr()))
    torch.cuda.synchronize()
    assert np.abs(dD.cpu().numpy() - want).max() <= 1e-4
