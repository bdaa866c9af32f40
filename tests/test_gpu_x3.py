"""GPU tier, kernel level: the fp32-accurate tensor-core GEMMs (csrc/gemm_x3.cu, 3 x tf32 wgmma on an
error-free hi / lo split) against an f64 reference.  Bound: a few 2^-22 of sum_k |a_k w_k| per output -- the accuracy class
of an f32 FMA chain (what the reference's ATen sgemm delivers on base.py:135-141), NOT tf32's 2^-11."""
import pytest
import torch

pytestmark = pytest.mark.gpu

REL = 1e-5          # worst element, of sum |terms| (measured 4e-6 at K = 672; an f32 FMA chain of that length: ~1e-6 typical)
REL_MEAN = 1e-6     # mean over the outputs


def _act(x, act):
    return {"none": x, "relu": torch.relu(x), "tanh": torch.tanh(x)}[act]


@pytest.mark.parametrize("R,K,N,ld_extra,bias,res,act,gather", [
    (1, 64, 64, 0, False, False, "none", False),
    (300, 300, 300, 20, True, True, "relu", False),
    (1000, 600, 600, 40, False, True, "relu", False),
    (777, 672, 600, 0, True, False, "tanh", False),
    (513, 372, 300, 0, True, False, "relu", True),
    (4100, 600, 600, 40, False, False, "none", False),
    (260, 32, 24, 0, False, False, "none", False),
])
def test_linear_x3_vs_f64(R, K, N, ld_extra, bias, res, act, gather):
    from chemprop_b200 import _lib, engine

    torch.manual_seed(R + K + N)
    dev = "cuda"
    src_rows = R + 50 if gather else R
    A = torch.zeros(src_rows, K + ld_extra, device=dev)
    A[:, :K] = torch.randn(src_rows, K, device=dev) * torch.rand(src_rows, 1, device=dev) * 3
    W = torch.randn(N, K, device=dev) / K ** 0.5
    b = torch.randn(N, device=dev) if bias else None
    ldc = (N + 63) // 64 * 64
    Rres = torch.zeros(R, ldc, device=dev)
    if res:
        Rres[:, :N] = torch.randn(R, N, device=dev)
    idx = torch.randint(0, src_rows, (R,), device=dev, dtype=torch.int32) if gather else None
    out = torch.full((R, ldc), 7.0, device=dev)
    code = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    engine.linear_x3(A, K, engine.pack_weight_x3(W), N, out, idx=idx, bias=b, res=Rres if res else None, act=code, R=R, pad_to=ldc)
    torch.cuda.synchronize()
    Ad = (A[idx.long()] if gather else A)[:, :K].double()
    Z = Ad @ W.double().t()
    if bias:
        Z = Z + b.double()
    if res:
        Z = Z + Rres[:, :N].double()
    ref = _act(Z, act)
    mag = Ad.abs() @ W.double().abs().t() + (Rres[:, :N].double().abs() if res else 0) + 1e-3
    err = (out[:, :N].double() - ref).abs()
    assert (err / mag).max().item() <= REL and (err / mag).mean().item() <= REL_MEAN, ((err / mag).max().item(), (err / mag).mean().item())
    n16 = min(ldc, (N + 15) // 16 * 16)
    assert float(out[:, N:n16].abs().max()) == 0.0 if n16 > N else True      # padding columns written as zeros
    if ldc > n16:
        assert bool((out[:, n16:] == 7.0).all())                                # ... and nothing beyond pad16(N) is touched


def test_linear_x3_transposed_weight_view():
    """dX = dY . W with W given as a column slice of a wider weight (W_o[:, d_v:], base.py:180): packed with transpose."""
    from chemprop_b200 import engine

    torch.manual_seed(0)
    Wo = torch.randn(300, 372, device="cuda") / 19
    dY = torch.zeros(900, 320, device="cuda")
    dY[:, :300] = torch.randn(900, 300, device="cuda")
    out = torch.zeros(900, 320, device="cuda")
    engine.linear_x3(dY, 300, engine.pack_weight_x3(Wo[:, 72:], transpose=True), 300, out, R=900, pad_to=320)
    ref = dY[:, :300].double() @ Wo[:, 72:].double()
    mag = dY[:, :300].double().abs() @ Wo[:, 72:].double().abs() + 1e-3
    assert (((out[:, :300].double() - ref).abs()) / mag).max().item() <= REL


@pytest.mark.parametrize("R,N,K,accumulate", [(1, 64, 64, False), (31, 300, 372, False), (5000, 600, 600, True),
                                              (2600, 600, 672, False), (70000, 300, 300, False), (33, 24, 32, True)])
def test_wgrad_x3_vs_f64(R, N, K, accumulate):
    from chemprop_b200 import engine

    torch.manual_seed(R + N + K)
    dev = "cuda"
    ldy, ldx = (N + 63) // 64 * 64, K + 8
    dY = torch.zeros(R, ldy, device=dev)
    dY[:, :N] = torch.randn(R, N, device=dev)
    X = torch.zeros(R, ldx, device=dev)
    X[:, :K] = torch.randn(R, K, device=dev) * torch.rand(R, 1, device=dev)
    dW0 = torch.randn(N, K, device=dev)
    dW = dW0.clone()
    engine.wgrad_x3(dY, X, R, N, K, dW, accumulate=accumulate)
    torch.cuda.synchronize()
    ref = dY[:, :N].double().t() @ X[:, :K].double() + (dW0.double() if accumulate else 0)
    mag = dY[:, :N].double().abs().t() @ X[:, :K].double().abs() + 1.0
    err = (dW.double() - ref).abs()
    assert (err / mag).max().item() <= REL and (err / mag).mean().item() <= REL_MEAN, ((err / mag).max().item(), (err / mag).mean().item())


def test_x3_is_deterministic():
    from chemprop_b200 import engine

    torch.manual_seed(3)
    dY, X = torch.randn(9000, 300, device="cuda"), torch.randn(9000, 300, device="cuda")
    a, b = torch.empty(300, 300, device="cuda"), torch.empty(300, 300, device="cuda")
    engine.wgrad_x3(dY, X, 9000, 300, 300, a)
    engine.wgrad_x3(dY, X, 9000, 300, 300, b)
    assert torch.equal(a, b)
