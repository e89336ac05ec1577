"""GPU: the DMMA NT GEMM at k-step counts around the 5-stage shared-memory ring of the TMA loader (K/16 = 1, 2, 4, 5,
6, 10, 11).  The TMA consumers load the first fragments of k-step s+1 while k-step s finishes and hand a ring slot back
only after that, so the first, the last, and the first wrapped k-steps are the cases that can go wrong.  Both loaders
run the same MMAs in the same order: they must agree bitwise, and match cuBLAS (torch.matmul, float64)."""
import pytest

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("K", [16, 32, 64, 80, 96, 160, 176])
def test_dgemm_nt_ring_lengths(engine, K):
    import torch
    torch.manual_seed(K)
    M, N = 384, 256
    A = torch.randn(M, K, dtype=torch.float64, device="cuda:0")
    B = torch.randn(N, K, dtype=torch.float64, device="cuda:0")
    C0 = torch.randn(M, N, dtype=torch.float64, device="cuda:0")
    C1 = C0.clone()
    ref = -(A @ B.T) + C0
    scale = float((A.abs() @ B.abs().T).max()) + float(C0.abs().max())
    engine.dgemm_nt_device(0, M, N, K, -1.0, A.data_ptr(), K, B.data_ptr(), K, 1.0, C0.data_ptr(), N)
    engine.dgemm_nt_device(1, M, N, K, -1.0, A.data_ptr(), K, B.data_ptr(), K, 1.0, C1.data_ptr(), N)
    torch.cuda.synchronize()
    assert torch.equal(C0, C1)
    assert float((C0 - ref).abs().max()) <= 2e-14 * scale
