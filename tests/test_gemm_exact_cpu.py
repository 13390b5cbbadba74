"""CPU side of the bit-exact GEMM tests (tests/exact_gemm.py): the exactness budget, its independence of summation
order, the CPU stand-ins of the binding against the fp64 reference with zero tolerance (a reduced-M copy of the GPU
matrix), the quantizers' rounding ties, and the stand-ins' refusal of wrong-shaped optional GEMM operands."""
import pytest
import torch

from tests import exact_gemm as X
from tests import fake_osb200 as F_
from tests.exact_gemm import quant_edge_rows, quant_expected

E4M3 = torch.float8_e4m3fn
CPU_M = 65
CASES = X.matrix(max_m=CPU_M)


def _standin(case):
    return getattr(F_, case.fn)


def test_budget_holds_for_every_case():
    """Every generator checks its case on construction; building the whole GPU matrix (M capped) must not raise."""
    assert len(CASES) > 150
    for idx, (name, builder, args, kw) in enumerate(CASES):
        builder(*args, seed=idx, **kw)


def test_budget_rejects_a_scale_off_the_power_of_two_grid():
    case = X.fp8_case(65, 72, 256, seed=1)
    case.a_scale = case.a_scale.clone()
    case.a_scale[7] = 3 * 2.0 ** -3
    with pytest.raises(X.BudgetError, match="a_scale"):
        X.check_budget(case)


def test_budget_rejects_an_fp8_partial_of_257():
    case = X.fp8_case(4, 8, 128, seed=2)
    case.a8 = torch.ones(4, 128).to(E4M3)
    w = torch.full((8, 128), 2.0)
    w[3, 5] = 3.0                       # row 3: 127 x 2 + 3 = 257
    case.w8 = w.to(E4M3)
    assert float((case.a8.double() @ case.w8.double().t()).max()) == 257
    with pytest.raises(X.BudgetError, match="FP8 k-block partial"):
        X.check_budget(case)


def test_budget_rejects_bf16_sums_past_22_bits():
    case = X.gemm_case(8, 8, 128, seed=3)
    case.a = torch.full((8, 128), 2.0 ** 12, dtype=torch.bfloat16)
    case.w = torch.full((8, 128), 2.0 ** 2, dtype=torch.bfloat16)
    with pytest.raises(X.BudgetError, match="bias"):   # 2^21 sums with a 2^-2 bias grid: 23 bits
        X.check_budget(case)


@pytest.mark.parametrize("idx", [0, 17, 45, 101, 150])
def test_summation_order_does_not_matter(idx):
    """On exact operands, fp32 matmul and a reversed chunked fp32 sum give the bits of the fp64 reference."""
    name, builder, args, kw = CASES[idx]
    case = builder(*args, seed=idx, **kw)
    if case.fn in ("gemm", "gemm_lora"):
        a, w = case.a.float(), case.w.float()
    else:   # fold the (power-of-two) scales in: exact
        sa = case.a_scale
        a = case.a8.float() * (sa.repeat_interleave(128, 1) if sa.dim() == 2 else sa[:, None])
        w = case.w8.float() * case.w_scale[:, None]
    want = a.double() @ w.double().t()
    fwd = a @ w.t()
    rev = torch.zeros_like(fwd)
    K = a.shape[1]
    for k0 in reversed(range(0, K, 8)):
        rev = rev + a[:, k0:k0 + 8] @ w[:, k0:k0 + 8].t()
    for got in (fwd, rev):
        X.assert_bits(f"{name} fp32", got, want.float())


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0] for c in CASES])
def test_standin_bit_identical(idx):
    name, builder, args, kw = CASES[idx]
    case = builder(*args, seed=idx, **kw)
    got = case.run(_standin(case))
    if case.epilogue == X.EPI_BIAS_GELU_TANH_FP8:
        want_codes, want_scales = X.fp8_gelu_expected(case.expected)
        X.assert_bits(f"{case} scales", got[1], want_scales)
        X.assert_bits(f"{case} codes", got[0], want_codes)
        assert bool((case.out_buf[:, :128] == 0x5A).all()) and bool((case.out_buf[:, 128 + case.N:] == 0x5A).all())
        assert bool((case.scale_buf[:, 0] == -7.0).all()) and bool((case.scale_buf[:, 1 + case.N // 128:] == -7.0).all())
    else:
        X.assert_bits(str(case), got, case.expected.to(torch.bfloat16))


# the row's amax is 448, so s = 1: round-to-nearest-even ties, normal and subnormal, the largest code and -0
TIE_CODES = [(1.0625, 0x38), (1.1875, 0x3A), (2.0 ** -10, 0x00), (3 * 2.0 ** -10, 0x02), (5 * 2.0 ** -10, 0x02),
             (448.0, 0x7E), (-0.0, 0x80)]


@pytest.mark.parametrize("which", ["rows", "blocks128", "blocksK"])
def test_quantizer_tie_table(which):
    x = quant_edge_rows()
    K = x.shape[1]
    if which == "rows":
        q, s = F_.quant_rows_fp8(x)
    else:
        q, s = F_.quant_blocks_fp8(x, block=128 if which == "blocks128" else K)
    codes = q.view(torch.uint8)
    assert [int(c) for c in codes[0, :len(TIE_CODES)]] == [c for _, c in TIE_CODES]
    assert [float(v) for v in x[0, :len(TIE_CODES)]] == [v for v, _ in TIE_CODES]
    assert bool((codes[1] == 0x80).all()), "an all -0 row keeps its sign"
    assert float(s.view(-1, s.shape[-1] if s.dim() == 2 else 1)[3, 0]) == 2.0 ** -4
    wq, ws = quant_expected(x, K if which == "rows" else (128 if which == "blocks128" else K))
    X.assert_bits(which, q, wq, signed_zero=True)
    X.assert_bits(which, s if s.dim() == 2 else s[:, None], ws, signed_zero=True)


def _views():
    """Wrong-shaped optional operands, each a view into a larger allocation."""
    b = lambda *s: torch.zeros(*s, dtype=torch.bfloat16)  # noqa: E731
    f = lambda *s: torch.zeros(*s, dtype=torch.float32)  # noqa: E731
    return b, f


@pytest.mark.parametrize("what", ["out", "bias", "residual", "gate_cols", "gate_rows", "mod_index", "k_mismatch"])
@pytest.mark.parametrize("fn", ["gemm", "gemm_lora", "dora", "gemm_fp8", "gemm_fp8_blocks"])
def test_standin_refuses_wrong_shapes(fn, what):
    b, f = _views()
    M, N, K = 16, 16, 128
    kw = dict(epilogue=X.EPI_BIAS_GATE_RES, residual=b(M, N), gate=f(2, N), group_rows=8)
    bias = b(N)
    if what == "out":
        kw["out"] = b(M, N)[:, :N - 8]
    elif what == "bias":
        bias = b(N)[:N - 8]
    elif what == "residual":
        kw["residual"] = b(M, N)[:M - 1]
    elif what == "gate_cols":
        kw["gate"] = f(2, N)[:, :N - 8]
    elif what == "gate_rows":
        kw["gate"] = f(2, N)[:1]
    elif what == "mod_index":
        kw["mod_index"] = torch.zeros(2, dtype=torch.int32)[:1]
    Kw = K + 128 if what == "k_mismatch" else K
    bf = fn in ("gemm", "gemm_lora", "dora")
    a = b(M, K) if bf else b(M, K).to(E4M3)
    w = b(N, Kw) if bf else b(N, Kw).to(E4M3)
    call = {
        "gemm": lambda: F_.gemm(a, w, bias, **kw),
        "gemm_lora": lambda: F_.gemm_lora(a, w, bias, b(M, 8), b(N, 8), **kw),
        "dora": lambda: F_.gemm_lora(a, w, bias, b(M, 8), b(N, 8), col_scale=torch.ones(N), **kw),
        "gemm_fp8": lambda: F_.gemm_fp8(a, torch.ones(M), w, torch.ones(N), bias, **kw),
        "gemm_fp8_blocks": lambda: F_.gemm_fp8_blocks(a, torch.ones(M, K // 128), w, torch.ones(N), bias, **kw),
    }[fn]
    n0 = F_.launch_count()
    with pytest.raises(F_.OsbError):
        call()
    assert F_.launch_count() == n0
