"""wgmma 3xTF32 forward (csrc/tc_gemm.cu) vs a float64 reference and vs the fp32 FFMA kernel.
Tolerance: max |err| <= 1e-5 * max(1, K/512) * max|y| (fp32-grade: three TF32 products recover ~22 mantissa bits;
the tensor core's fp32 accumulation error grows linearly with the contraction length: 4e-6 at K=512, 1.6e-5 at
K=3136 — both far inside the 1e-4 learner tolerance)."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("M,N,K", [(128, 128, 32), (1024, 512, 512), (4096, 512, 512), (16384, 512, 512), (2048, 128, 3136 - 3136 % 32)])
@pytest.mark.parametrize("relu", [0, 1])
def test_tc_linear_fwd(M, N, K, relu):
    from jorldy_b200._lib import C
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g).cuda()
    w = (torch.randn(N, K, generator=g) / K ** 0.5).cuda()
    b = torch.randn(N, generator=g).cuda()
    y = torch.full((M, N), float("nan"), device="cuda")
    s = torch.cuda.current_stream().cuda_stream
    C.jb_linear_fwd_tc(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), M, K, N, relu, s)
    y2 = torch.empty(M, N, device="cuda")
    C.jb_linear_fwd(x.data_ptr(), w.data_ptr(), b.data_ptr(), y2.data_ptr(), M, K, N, relu, s)
    torch.cuda.synchronize()
    ref = x.double() @ w.double().t() + b.double()
    if relu:
        ref = torch.relu(ref)
    scale = ref.abs().max().item()
    assert not torch.isnan(y).any()
    e1, e2 = (y.double() - ref).abs().max().item(), (y - y2).abs().max().item()
    tol = 1e-5 * max(1.0, K / 512) * scale
    assert e1 <= tol, (e1, scale)
    assert e2 <= tol, (e2, scale)


def test_tc_rejects_unsupported_shapes():
    from jorldy_b200._lib import JbError, C
    x = torch.zeros(100, 64, device="cuda"); w = torch.zeros(128, 64, device="cuda"); b = torch.zeros(128, device="cuda")
    y = torch.zeros(100, 128, device="cuda")
    with pytest.raises(JbError):
        C.jb_linear_fwd_tc(x.data_ptr(), w.data_ptr(), b.data_ptr(), y.data_ptr(), 100, 64, 128, 0, 0)
