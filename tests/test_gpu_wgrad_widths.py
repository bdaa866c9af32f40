"""GPU tier: k_wgrad_tc at every accumulator width it instantiates, against float64.

A CTA of k_wgrad_tc issues one wgmma m64n{kw}k16 per k16 step, kw = the 16, 32, ..., 192 output columns of its column tile
(csrc/wgrad_tc.cu), and a warpgroup whose 64 output rows lie beyond N does not run.  Each width is its own instruction
shape with its own B descriptor span.  The cases here run every width as the only column tile and as the second one behind a
192-column tile, with one, two and three dY terms, with one and with two working warpgroups in the last row tile, and with
several row blocks per CTA so that the in-flight group of one block overlaps the next.

Operands are integer-valued, so every partial sum is an integer below 2^24 and the f32 accumulator is exact in any order:
dW must equal the float64 reference bit for bit.  NaN fills every operand column past N / K and every row past R."""
import pytest
import torch

pytestmark = pytest.mark.gpu

NAN = float("nan")
R = 40_000              # 625 row blocks: four or more per CTA at 132 row slots


def _operand(g, rows, cols):
    t = torch.full((rows + 5, (cols + 7) // 8 * 8 + 8), NAN, dtype=torch.bfloat16, device="cuda")
    t[:rows, :cols] = torch.randint(-2, 3, (rows, cols), device="cuda", generator=g).bfloat16()
    return t


CASES = [(w - 3, (40, 300, 200)[i % 3], 1 + i % 3) for i, w in enumerate(range(16, 193, 16))]      # one column tile
CASES += [(192 + w - 3, (300, 129)[i % 2], 1) for i, w in enumerate(range(16, 193, 16))]           # 192 columns + w


@pytest.mark.parametrize("K,N,n_terms", CASES)
def test_wgrad_tc_every_width_exact(K, N, n_terms):
    from chemprop_b200.engine import wgrad_tc, wgrad_tc_multi

    g = torch.Generator(device="cuda").manual_seed(1000 * K + N)
    dYs = [_operand(g, R, N) for _ in range(n_terms)]
    X = _operand(g, R, K)
    dW = torch.full((N, K), NAN, device="cuda")
    if n_terms == 1:
        wgrad_tc(dYs[0], X, R, N, K, dW)
    else:
        wgrad_tc_multi(dYs, X, R, N, K, dW)
    torch.cuda.synchronize()
    ref = sum(t[:R, :N].double().t() @ X[:R, :K].double() for t in dYs)
    assert float(ref.abs().max()) < (1 << 24)
    assert torch.equal(dW.double(), ref), (K, N, n_terms, float((dW.double() - ref).abs().max()))
