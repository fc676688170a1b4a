"""Dense-layer kernels vs a float64-accumulated torch reference over the shapes and operand layouts
the networks use, including ragged sizes that exercise the generic (non-cp.async) path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

SHAPES = [(256, 512, 512), (32, 512, 512), (2048, 512, 512), (256, 512, 4), (256, 2, 512), (100, 130, 77),
          (4096, 512, 512), (33, 204, 512), (256, 512, 3136), (17, 64, 64),
          # launch_gemm takes the 128x64 tile once ceil(M/128) * ceil(N/64) >= 264; these are the products that reach it
          (204800, 32, 256),   # conv1 at B=512 (M = B*20*20): forward (half-empty N tile) and dx
          (41472, 64, 512),    # conv2 at B=512 (M = B*9*9): forward and dx
          (25088, 64, 576),    # conv3 at B=512 (M = B*7*7): dx only (its forward is 196 tiles)
          (40001, 33, 130),    # ragged M and N = 33 < 64: forward and dx
          (512, 2048, 2048)]   # dw only, in the (0, 0) layout with the row-sum (db) epilogue


def _ref(a, b):
    return (a.double() @ b.double()).float()


def _dw_atol(M):
    """dw / db contract over the M rows.  2e-4 * sqrt(M / 256) holds while the contraction is cut into short chains;
    one fp32 chain of M unit-variance products has a rounding error of std <= u*M/sqrt(6) (u = 2^-24: each partial
    sum s_k has E[s_k^2] = k and rounds by at most u|s_k|), so long contractions get 6 of those standard deviations."""
    return max(2e-4 * max(1.0, M / 256) ** 0.5, 6 * 2.0 ** -24 * M / 6 ** 0.5)


@pytest.mark.parametrize("M,N,K", SHAPES)
def test_linear_fwd_bwd(M, N, K):
    from jorldy_b200.core.network import layers as L
    g = torch.Generator().manual_seed(M * 7 + N * 3 + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    xd, wd, bd, dyd = x.cuda(), w.cuda(), b.cuda(), dy.cuda()
    y = torch.empty(M, N, device="cuda")
    L.linear_fwd(xd, wd, bd, y, relu=True)
    ref = torch.relu(_ref(x, w.t()) + b)
    np.testing.assert_allclose(y.cpu().numpy(), ref.numpy(), rtol=2e-5, atol=2e-5)
    act = torch.relu(torch.randn(M, K, generator=g))
    dx = torch.empty(M, K, device="cuda")
    L.linear_bwd_dx(dyd, wd, dx, relu_act=act.cuda())
    np.testing.assert_allclose(dx.cpu().numpy(), (_ref(dy, w) * (act > 0)).numpy(), rtol=2e-5, atol=5e-5)
    dw = torch.empty(N, K, device="cuda")
    db = torch.empty(N, device="cuda")
    L.linear_bwd_dw(dyd, xd, dw, db)
    np.testing.assert_allclose(dw.cpu().numpy(), _ref(dy.t(), x).numpy(), rtol=2e-5, atol=_dw_atol(M))
    np.testing.assert_allclose(db.cpu().numpy(), dy.double().sum(0).float().numpy(), rtol=2e-5, atol=_dw_atol(M))


@pytest.mark.parametrize("M,N,K", [(256, 512, 512), (32, 204, 512), (64, 51, 512), (100, 130, 76)])
def test_linear_io_fwd_bwd(M, N, K):
    """NoisyNet layout: weight [in, out], y = x @ W + b (network/utils.py:84)."""
    from jorldy_b200.core.network import layers as L
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g)
    w = torch.randn(K, N, generator=g) / K ** 0.5
    b = torch.randn(N, generator=g)
    dy = torch.randn(M, N, generator=g)
    xd, wd, bd, dyd = x.cuda(), w.cuda(), b.cuda(), dy.cuda()
    y = torch.empty(M, N, device="cuda")
    L.linear_io_fwd(xd, wd, bd, y, relu=False)
    np.testing.assert_allclose(y.cpu().numpy(), (_ref(x, w) + b).numpy(), rtol=2e-5, atol=2e-5)
    dx = torch.empty(M, K, device="cuda")
    L.linear_io_bwd_dx(dyd, wd, dx)
    np.testing.assert_allclose(dx.cpu().numpy(), _ref(dy, w.t()).numpy(), rtol=2e-5, atol=5e-5)
    dw = torch.empty(K, N, device="cuda")
    db = torch.empty(N, device="cuda")
    L.linear_io_bwd_dw(dyd, xd, dw, db)
    np.testing.assert_allclose(dw.cpu().numpy(), _ref(x.t(), dy).numpy(), rtol=2e-5, atol=2e-4)
    np.testing.assert_allclose(db.cpu().numpy(), dy.double().sum(0).float().numpy(), rtol=2e-5, atol=2e-4)


def test_gemm_row_position_independence():
    """A row's forward result does not depend on where it sits in the batch (needed by the PPO
    value-shift pre-pass and by minibatch-vs-full-batch parity)."""
    from jorldy_b200.core.network import layers as L
    g = torch.Generator().manual_seed(0)
    x = torch.randn(300, 512, generator=g).cuda()
    w = torch.randn(512, 512, generator=g).cuda()
    b = torch.zeros(512).cuda()
    y = torch.empty(300, 512, device="cuda")
    L.linear_fwd(x, w, b, y, relu=False)
    perm = torch.randperm(300, generator=g).cuda()
    xp = x[perm].contiguous()
    yp = torch.empty(300, 512, device="cuda")
    L.linear_fwd(xp, w, b, yp, relu=False)
    assert torch.equal(y[perm], yp)
    y1 = torch.empty(37, 512, device="cuda")
    L.linear_fwd(x[:37].contiguous(), w, b, y1, relu=False)
    assert torch.equal(y[:37], y1)


@pytest.mark.parametrize("M,N,K,splits", [(12800, 32, 256, 37), (2592, 64, 512, 5), (1568, 64, 576, 3), (5003, 33, 130, 8)])
def test_linear_bwd_dw_splitk(M, N, K, splits):
    """Conv-layer weight gradients (tiny [out, in] output, contraction over batch x positions) through the grid-level
    split-K kernel + fixed-order fold: equal to the float64 reference and bit-reproducible."""
    from jorldy_b200.core.dev import C, ptr, stream_ptr
    g = torch.Generator().manual_seed(M + N + K)
    x = torch.randn(M, K, generator=g)
    dy = torch.randn(M, N, generator=g)
    xd, dyd = x.cuda(), dy.cuda()
    ws = torch.empty(splits * (N * K + N), device="cuda")
    out = []
    for _ in range(2):
        dw = torch.full((N, K), float("nan"), device="cuda")
        db = torch.full((N,), float("nan"), device="cuda")
        C.jb_linear_bwd_dw_splitk(ptr(dyd), ptr(xd), ptr(dw), ptr(db), M, K, N, ptr(ws), splits, stream_ptr())
        out.append((dw.cpu(), db.cpu()))
    tol = 2e-4 * max(1.0, M / 256) ** 0.5
    np.testing.assert_allclose(out[0][0].numpy(), _ref(dy.t(), x).numpy(), rtol=2e-5, atol=tol)
    np.testing.assert_allclose(out[0][1].numpy(), dy.double().sum(0).float().numpy(), rtol=2e-5, atol=tol)
    assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
