"""GPU tier: the wgmma linear kernel (dmpnn_linear_tc_bf16) and its helpers against a plain PyTorch
fp32 reference of the same op (bf16 operands, fp32 accumulate)."""
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(A, K, W, b, act):
    z = A[:, :K].float() @ W.bfloat16().float().t()
    if b is not None:
        z = z + b
    return {"none": lambda x: x, "relu": torch.relu, "tanh": torch.tanh}[act](z)


@pytest.mark.parametrize("R,K,lda,N,act,bias", [
    (1000, 86, 96, 300, "none", False), (5000, 300, 320, 300, "none", False), (3000, 372, 384, 300, "relu", True),
    (128, 64, 64, 64, "tanh", True), (37, 16, 16, 16, "relu", False), (20000, 300, 320, 300, "relu", True),
    (257, 300, 304, 256, "none", True), (513, 200, 208, 304, "relu", False),
])
def test_linear_tc_vs_torch(R, K, lda, N, act, bias):
    from chemprop_b200 import _lib
    from chemprop_b200.engine import linear_tc, pack_weight_tc

    g = torch.Generator(device="cuda").manual_seed(R + K)
    A = torch.zeros(R, lda, dtype=torch.bfloat16, device="cuda")
    A[:, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    if lda > K:
        A[:, K:] = 7.0          # garbage beyond K must be ignored (TMA clips at the tensor's inner extent)
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1 if bias else None
    Np = (N + 15) // 16 * 16
    ldc = (Np + 63) // 64 * 64
    out = torch.full((R, ldc), float("nan"), dtype=torch.bfloat16, device="cuda")
    code = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    linear_tc(A, K, pack_weight_tc(W), N, out, bias=b, act=code)
    torch.cuda.synchronize()
    ref = _ref(A, K, W, b, act)
    assert torch.isfinite(out[:, :Np].float()).all()
    torch.testing.assert_close(out[:, :N].float(), ref.bfloat16().float(), rtol=2 ** -7, atol=2e-3)
    if Np > N:
        assert float(out[:, N:Np].float().abs().max()) == 0.0
    if ldc > Np:
        assert torch.isnan(out[:, Np:].float()).all()       # columns beyond pad16(N) are never touched


def test_linear_tc_transposed_weight_slice():
    """dX = dY . W_o[:, d_v:]  ->  B[n][k] = W[k][d_v + n]  (transpose packing of a column slice)."""
    from chemprop_b200.engine import linear_tc, pack_weight_tc

    torch.manual_seed(0)
    h, d_v, R = 300, 72, 4000
    Wo = torch.randn(h, d_v + h, device="cuda") / (d_v + h) ** 0.5
    dY = torch.zeros(R, 320, dtype=torch.bfloat16, device="cuda")
    dY[:, :h] = torch.randn(R, h, device="cuda").bfloat16()
    out = torch.zeros(R, 320, dtype=torch.bfloat16, device="cuda")
    linear_tc(dY, h, pack_weight_tc(Wo[:, d_v:], transpose=True), h, out)
    ref = dY[:, :h].float() @ Wo[:, d_v:].bfloat16().float()
    torch.testing.assert_close(out[:, :h].float(), ref.bfloat16().float(), rtol=2 ** -7, atol=2e-3)


def test_concat_bf16():
    from chemprop_b200.engine import concat_bf16

    torch.manual_seed(1)
    V = torch.randn(50, 72, device="cuda")
    E = torch.randn(120, 14, device="cuda")
    i1 = torch.randint(0, 50, (120,), device="cuda", dtype=torch.int32)
    i2 = torch.randperm(120, device="cuda").to(torch.int32)
    out = torch.full((120, 96), float("nan"), dtype=torch.bfloat16, device="cuda")
    concat_bf16(V, 72, out, 120, idx1=i1, X2=E, K2=14, idx2=i2)
    ref = torch.cat([V[i1.long()], E[i2.long()], torch.zeros(120, 10, device="cuda")], 1).bfloat16()
    assert torch.equal(out, ref)


@pytest.mark.parametrize("R,N,K,lddy,ldx", [
    (5000, 300, 300, 320, 320), (3000, 300, 86, 320, 96), (2500, 300, 372, 320, 384), (64, 64, 64, 64, 64),
    (1, 300, 300, 320, 320), (200000, 300, 300, 320, 320), (777, 128, 16, 128, 16),
])
def test_wgrad_tc_vs_torch(R, N, K, lddy, ldx):
    from chemprop_b200.engine import wgrad_tc

    g = torch.Generator(device="cuda").manual_seed(R + K)
    dY = torch.full((R, lddy), 3.0, dtype=torch.bfloat16, device="cuda")     # garbage beyond N / K must be ignored
    dY[:, :N] = torch.randn(R, N, device="cuda", generator=g).bfloat16()
    X = torch.full((R, ldx), -2.0, dtype=torch.bfloat16, device="cuda")
    X[:, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    dW = torch.full((N, K), 0.5, device="cuda")
    ref = dY[:, :N].double().t() @ X[:, :K].double()
    wgrad_tc(dY, X, R, N, K, dW)
    torch.cuda.synchronize()
    scale = max(1.0, float(ref.abs().max()))
    assert (dW.double() - ref).abs().max().item() <= 2e-4 * scale * max(1.0, (R / 1000) ** 0.5)
    wgrad_tc(dY, X, R, N, K, dW, accumulate=True)
    assert (dW.double() - 2 * ref).abs().max().item() <= 4e-4 * scale * max(1.0, (R / 1000) ** 0.5)


@pytest.mark.parametrize("R,N,K,lddy,ldx,n_terms", [
    (5000, 300, 147, 304, 160, 3), (3000, 300, 300, 320, 320, 2), (2500, 300, 372, 320, 384, 3), (130, 64, 64, 64, 64, 3),
    (200000, 300, 147, 304, 152, 3), (700, 300, 133, 304, 136, 5),
])
def test_wgrad_tc_multi_term(R, N, K, lddy, ldx, n_terms):
    """dW = sum_t dY_t^T X with the terms sharing the X stream (dmpnn_wgrad_tc_multi_bf16): equals the sum of the
    single-term results up to f32 summation order; term lists longer than a stage holds are issued in groups."""
    from chemprop_b200.engine import wgrad_tc_multi

    g = torch.Generator(device="cuda").manual_seed(R + K + n_terms)
    dYs = []
    for _ in range(n_terms):
        dY = torch.full((R, lddy), 3.0, dtype=torch.bfloat16, device="cuda")
        dY[:, :N] = torch.randn(R, N, device="cuda", generator=g).bfloat16()
        dYs.append(dY)
    X = torch.full((R, ldx), -2.0, dtype=torch.bfloat16, device="cuda")
    X[:, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    ref = sum(dY[:, :N].double().t() @ X[:, :K].double() for dY in dYs)
    dW = torch.full((N, K), 0.5, device="cuda")
    wgrad_tc_multi(dYs, X, R, N, K, dW)
    torch.cuda.synchronize()
    scale = max(1.0, float(ref.abs().max()))
    tol = 2e-4 * scale * max(1.0, (n_terms * R / 1000) ** 0.5)
    assert (dW.double() - ref).abs().max().item() <= tol
    wgrad_tc_multi(dYs, X, R, N, K, dW, accumulate=True)
    assert (dW.double() - 2 * ref).abs().max().item() <= 2 * tol
    dW2 = torch.empty_like(dW)
    wgrad_tc_multi(dYs, X, R, N, K, dW2)
    wgrad_tc_multi(dYs, X, R, N, K, dW)
    assert torch.equal(dW, dW2)                      # deterministic


@pytest.mark.parametrize("R,C,ld,gather", [(5000, 304, 304, True), (4097, 300, 304, False), (333, 64, 64, True), (7, 300, 320, True),
                                           (100000, 304, 304, True)])
def test_act_bwd_relu_bf16_fast_path(R, C, ld, gather):
    """All-bf16 ReLU instance of dmpnn_act_bwd (packed-pair mask kernel): dZ[r] = G[gidx[r]] where Y[r] > 0, else 0 --
    bit-exact, including y = 0, y = -0 and NaN (no gradient)."""
    from chemprop_b200.engine import ACT_RELU, act_bwd

    g = torch.Generator(device="cuda").manual_seed(R + C)
    nG = R // 2 + 1 if gather else R
    G = torch.randn(nG, ld, device="cuda", generator=g).bfloat16()
    Y = torch.randn(R, ld, device="cuda", generator=g).bfloat16()
    Y[::7, ::3] = 0.0
    Y[1::7, 1::3] = -0.0
    Y[2::11, 2::5] = float("nan")
    gidx = torch.randint(0, nG, (R,), device="cuda", dtype=torch.int32, generator=g) if gather else None
    dZ = torch.full((R, ld), 9.0, dtype=torch.bfloat16, device="cuda")
    act_bwd(G, Y, R, C, act=ACT_RELU, gidx=gidx, dZ=dZ)
    Gr = G[gidx.long()] if gather else G
    ref = torch.where(Y[:, :C] > 0, Gr[:, :C], torch.zeros((), dtype=torch.bfloat16, device="cuda"))
    assert torch.equal(dZ[:, :C], ref)
    assert bool((dZ[:, C:] == 9.0).all())                                 # nothing written beyond C
    dZ2 = torch.empty_like(dZ)
    act_bwd(G, Y, R, C, act=ACT_RELU, gidx=gidx, dZ=dZ2, from_preact=True)
    assert torch.equal(dZ2[:, :C], ref)


def test_column_sum():
    from chemprop_b200.engine import column_sum

    Y = torch.randn(70001, 320, device="cuda").bfloat16()
    out = torch.zeros(300, device="cuda")
    column_sum(Y, 70001, 300, out)
    torch.testing.assert_close(out, Y[:, :300].float().sum(0), rtol=1e-4, atol=1e-2)


@pytest.mark.parametrize("R,K,N,act", [(3000, 314, 300, "relu"), (130, 142, 128, "tanh"), (5000, 64, 64, "none")])
def test_linear_tc_residual(R, K, N, act):
    """C = act(A . W^T + b + res): the H_0 residual of the update (base.py:138) added in the GEMM epilogue
    (AtomMessagePassing's depth step on the tensor cores)."""
    from chemprop_b200 import _lib
    from chemprop_b200.engine import linear_tc, pack_weight_tc

    g = torch.Generator(device="cuda").manual_seed(R + K)
    lda = (K + 15) // 16 * 16
    A = torch.zeros(R, lda, dtype=torch.bfloat16, device="cuda")
    A[:, :K] = torch.randn(R, K, device="cuda", generator=g).bfloat16()
    W = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g) * 0.1
    ldc = (N + 63) // 64 * 64
    res = torch.zeros(R, ldc, dtype=torch.bfloat16, device="cuda")
    res[:, :N] = torch.randn(R, N, device="cuda", generator=g).bfloat16()
    out = torch.full((R, ldc), float("nan"), dtype=torch.bfloat16, device="cuda")
    code = {"none": _lib.ACT_NONE, "relu": _lib.ACT_RELU, "tanh": _lib.ACT_TANH}[act]
    linear_tc(A, K, pack_weight_tc(W), N, out, bias=b, res=res, act=code)
    torch.cuda.synchronize()
    z = A[:, :K].float() @ W.bfloat16().float().t() + b + res[:, :N].float()
    ref = {"none": lambda x: x, "relu": torch.relu, "tanh": torch.tanh}[act](z)
    torch.testing.assert_close(out[:, :N].float(), ref.bfloat16().float(), rtol=2 ** -7, atol=4e-3)
    with pytest.raises(Exception):
        linear_tc(A, K, pack_weight_tc(W), N, out, res=out)          # the residual may not alias the output
