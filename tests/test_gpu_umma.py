"""Known-answer test of the tensor-core plumbing (csrc/wgmma.cuh): one CTA of two warpgroups computes D[128, N] = A[128, K] . B[N, K]^T
with wgmma.mma_async (TF32 inputs, FP32 accumulators in registers) from K-major, unswizzled shared-memory operands.  The Leung-Malik
contraction (csrc/lm_texture.cu) uses exactly these operand layouts and descriptor encodings.

The module and test names come from the earlier tcgen05 version of the contraction; they are kept so that the same test ids check
the same shapes and tolerances, now through wgmma."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _tf32(x):
    bits = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((bits + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def _run(lib, torch, A, B, variant):
    from pyimsegm_b200 import _lib
    N, K = B.shape
    dA, dB = torch.from_numpy(A).cuda(), torch.from_numpy(B).cuda()
    dD = torch.zeros((128, N), dtype=torch.float32, device='cuda')
    _lib.check(lib.isb_wgmma_selftest(_lib.ptr(dA), _lib.ptr(dB), N, K, variant, _lib.ptr(dD), _lib.stream_ptr()))
    torch.cuda.synchronize()
    return dD.cpu().numpy()


@pytest.mark.parametrize('N,K', [(80, 40), (48, 40), (16, 8), (256, 64)])
def test_tcgen05_tf32_gemm_known_answer(N, K):
    from pyimsegm_b200 import _lib
    torch = _lib.require_cuda()
    lib = _lib.lib()
    rng = np.random.RandomState(N + K)
    A = _tf32(rng.standard_normal((128, K)).astype(np.float32))
    B = _tf32(rng.standard_normal((N, K)).astype(np.float32))
    want = A.astype(np.float64) @ B.astype(np.float64).T
    got = _run(lib, torch, A, B, 0)
    err = np.abs(got - want).max()
    if err > 1e-4:
        alt = np.abs(_run(lib, torch, A, B, 1) - want).max()
        raise AssertionError('wgmma GEMM wrong: max err %g (with LBO/SBO swapped: %g)' % (err, alt))


@pytest.mark.parametrize('N,K', [(80, 40), (48, 40), (240, 64)])
def test_tcgen05_tf32_gemm_a_operand_in_tensor_memory(N, K):
    """the A operand in the form the contraction feeds it: per-thread register fragments (there is no tensor memory on sm_90),
    B from shared memory"""
    from pyimsegm_b200 import _lib
    torch = _lib.require_cuda()
    lib = _lib.lib()
    rng = np.random.RandomState(7 * N + K)
    A = _tf32(rng.standard_normal((128, K)).astype(np.float32))
    B = _tf32(rng.standard_normal((N, K)).astype(np.float32))
    want = A.astype(np.float64) @ B.astype(np.float64).T
    got = _run(lib, torch, A, B, 2)
    assert np.abs(got - want).max() <= 1e-4
