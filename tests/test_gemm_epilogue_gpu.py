"""The staged GEMM epilogue's edges, bit for bit: outputs written by TMA tile stores into a view of a larger buffer, and the
implicit-GEMM convolution's 5-D output box clipped at the edges of the output.

- `gemm`, `gemm_lora` and `gemm_fp8` write into a column slice of a sentinel-filled buffer with extra columns on both
  sides and extra rows below (row stride > N, M not a multiple of 128, N not a multiple of the tile width), for every
  tile width and for the bias, GELU and gate + residual epilogues (modulation groups that straddle tiles, `mod_index`,
  output aliasing the residual).  The values must equal the exact fp64 reference rounded once (tests/exact_gemm.py) and
  no byte outside the view may change: a store map sized by the row stride or by the padded M would write there.
- `conv3d` with a residual, on exact operands, over an output whose extents are not multiples of the CTA's Wt x Ht x Tt
  box in any of t, h and w, and a channel count that leaves the last column tile mostly empty."""
import pytest
import torch

from tests import exact_gemm as X

pytestmark = pytest.mark.gpu

SENTINEL = -7.25          # bf16-exact, never produced by the cases below at these positions
PAD_ROWS = 5
M, N, K = 333, 520, 256   # 3 row tiles (the last with 77 rows); 520 columns: a ragged last tile at every width


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _in_sentinel_buffer(case):
    """Points case.out at rows [0, M) x columns [PAD, PAD + N) of a [M + PAD_ROWS, N + 2 PAD] sentinel buffer.  With
    out aliasing the residual, the residual's values move into that view too (the expected result is unchanged)."""
    pad = X.PAD // 2
    buf = torch.full((case.M + PAD_ROWS, case.N + 2 * pad), SENTINEL, dtype=torch.bfloat16, device=case.expected.device)
    view = buf[:case.M, pad:pad + case.N]
    if case.out is not None:     # "alias": out is the residual
        view.copy_(case.residual)
        case.residual = view
    case.out = view
    return buf, pad


def _cases():
    out = []
    epis = [(X.EPI_BIAS, None), (X.EPI_BIAS_GELU_TANH, None)] + [(X.EPI_BIAS_GATE_RES, g) for g in ("groups", "mod_index", "alias")]
    for bn in (64, 128, 192, 256):
        for epi, gm in epis:
            out.append(("gemm", bn, epi, gm))
        out.append(("lora", bn, X.EPI_BIAS_GATE_RES, "alias"))
        out.append(("lora", bn, X.EPI_BIAS_GATE_RES, "groups"))
    for bn in (64, 128):
        for epi, gm in ((X.EPI_BIAS, None), (X.EPI_BIAS_GATE_RES, "mod_index"), (X.EPI_BIAS_GATE_RES, "alias")):
            out.append(("fp8", bn, epi, gm))
    return out


CASES = _cases()


@pytest.mark.parametrize("fn,bn,epi,gm", CASES, ids=[f"{f}-bn{b}-{X.EPI_NAMES[e]}" + (f"-{g}" if g else "") for f, b, e, g in CASES])
def test_output_view_in_sentinel_buffer(fn, bn, epi, gm):
    import osb200 as osb

    dev = _dev()
    seed = CASES.index((fn, bn, epi, gm))
    if fn == "gemm":
        case = X.gemm_case(M, N, K, epi, gate_mode=gm, block_n=bn, seed=seed, device=dev)
    elif fn == "lora":
        case = X.lora_case(M, N, K, 72, epi, col_scale=True, gate_mode=gm, block_n=bn, seed=seed, device=dev)
    else:
        case = X.fp8_case(M, N, K, epi, gate_mode=gm, block_n=bn, seed=seed, device=dev)
    buf, pad = _in_sentinel_buffer(case)
    got = case.run(osb)
    torch.cuda.synchronize()
    assert got.data_ptr() == case.out.data_ptr()
    X.assert_bits(str(case), got, case.expected.to(torch.bfloat16))
    outside = buf.clone()
    outside[:M, pad:pad + N] = SENTINEL
    bad = (outside != SENTINEL).nonzero()
    assert bad.numel() == 0, f"{case}: wrote {bad.shape[0]} elements outside the output view, first at {tuple(bad[0].tolist())}"


@pytest.mark.parametrize("block_n", [128, 64])
def test_conv3d_residual_ragged_box(block_n):
    """3x3x3 convolution + bias + residual on exact operands (x in {0, +-1}, w in {0, +-1} x 2^e per output channel, bias
    and residual multiples of 2^-2): the output must equal the fp64 reference bit for bit, also where the CTA box hangs
    over the output's edge in t, h and w, and over the last channels."""
    import torch.nn.functional as F

    import osb200 as osb

    dev = _dev()
    nb, (t, h, w), cin, cout = 2, (3, 3, 12), 64, 136
    Tt, Ht, Wt = X.conv_box(t, h, w)
    assert t % Tt and h % Ht and w % Wt, f"box {Tt}x{Ht}x{Wt} is not ragged in every dimension of {t}x{h}x{w}"
    g = torch.Generator(device=dev).manual_seed(11)
    ints = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g, device=dev).double()   # noqa: E731
    x = ints(-1, 1, nb, t + 2, h + 2, w + 2, cin)
    wt = ints(-1, 1, cout, cin, 3, 3, 3) * torch.ldexp(torch.ones(cout, 1, 1, 1, 1, device=dev, dtype=torch.float64),
                                                       ints(-2, 2, cout, 1, 1, 1, 1).long())
    bias = ints(-256, 256, cout) / 4
    res = ints(-256, 256, nb, t, h, w, cout) / 4
    ref = F.conv3d(x.permute(0, 4, 1, 2, 3).cpu(), wt.cpu()).permute(0, 2, 3, 4, 1).to(dev) + bias + res
    assert float(ref.abs().max()) < 2.0 ** 20   # multiples of 2^-2: exact in fp32 and in the fp64 reference
    y = osb.conv3d(x.to(torch.bfloat16), osb.pack_conv_weight(wt.to(torch.bfloat16), 64, False), bias.to(torch.bfloat16),
                   out_thw=(t, h, w), residual=res.to(torch.bfloat16), block_n=block_n)
    torch.cuda.synchronize()
    X.assert_bits(f"conv3d {nb}x{t}x{h}x{w}x{cout} box {Tt}x{Ht}x{Wt} block_n {block_n}", y, ref.to(torch.bfloat16))
