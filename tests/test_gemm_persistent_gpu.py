"""GPU checks of the persistent schedule of gemm_bf16_kernel: one CTA per SM walks output tiles b, b + grid, ...,
carrying the stage ring across tiles and reusing one epilogue buffer.  Every case has more tiles than SMs, ragged M and
N, and k-block counts that are not a multiple of the stage count (K = 1152: 18 bf16 k-blocks against 3 / 4 / 6 stages;
K = 320: 5; K = 64: 1, fewer than the stages), on the exact operands of tests/exact_gemm.py: a tile mix-up, a stale
accumulator, a stale residual or an output stored over the next tile's residual changes the bits."""
import functools

import pytest
import torch

from tests import exact_gemm as X
from tests.util import read_tiles

pytestmark = pytest.mark.gpu

M = 12345                   # 97 row tiles, the last with 57 rows
N = 1096                    # 18 / 9 / 6 / 5 column tiles at block_n 64 / 128 / 192 / 256, the last one ragged
EPIS = [(X.EPI_BIAS, None), (X.EPI_BIAS_GELU_TANH, None), (X.EPI_BIAS_GATE_RES, "mod_index"),
        (X.EPI_BIAS_GATE_RES, "alias")]


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _tiles(M_, N_, bn):
    return -(-M_ // 128) * -(-N_ // bn)


def _check(case, bn):
    import osb200 as osb

    assert _tiles(case.M, case.N, bn) > 2 * _sms(), "the case must give every CTA several tiles"
    got = case.run(osb)
    torch.cuda.synchronize()
    if case.out is not None:
        assert got.data_ptr() == case.out.data_ptr()
    X.assert_bits(str(case), got, case.expected.to(torch.bfloat16))


@pytest.mark.parametrize("K", [1152, 320, 64])
@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("epi,gm", EPIS, ids=[X.EPI_NAMES[e] + (f"-{g}" if g else "") for e, g in EPIS])
def test_gemm_many_tiles(epi, gm, bn, K):
    dev = _dev()
    _check(X.gemm_case(M, N, K, epi, gate_mode=gm, block_n=bn, seed=bn + K + epi, device=dev), bn)


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("epi,gm", [(X.EPI_BIAS, None), (X.EPI_BIAS_GATE_RES, "alias")])
def test_lora_many_tiles(epi, gm, bn):
    """5 base k-blocks and 2 rank k-blocks per tile, DoRA's column scale."""
    dev = _dev()
    _check(X.lora_case(M, N, 320, 72, epi, col_scale=True, gate_mode=gm, block_n=bn, seed=bn, device=dev), bn)


@pytest.mark.parametrize("K", [1152, 640, 128])
@pytest.mark.parametrize("bn", [64, 128])
@pytest.mark.parametrize("fn", ["fp8", "fp8_blocks"])
@pytest.mark.parametrize("epi,gm", [(X.EPI_BIAS, None), (X.EPI_BIAS_GATE_RES, "alias")])
def test_fp8_many_tiles(epi, gm, fn, bn, K):
    """9 / 5 / 1 e4m3 k-blocks of 128 per tile."""
    dev = _dev()
    build = X.fp8_case if fn == "fp8" else X.fp8_blocks_case
    _check(build(M, N, K, epi, gate_mode=gm, block_n=bn, seed=bn + K, device=dev), bn)


def test_fp8_gelu_out_many_tiles():
    """The FP8-emitting GELU epilogue goes on to the CTA's next tile instead of ending the CTA."""
    import osb200 as osb

    dev = _dev()
    case = X.fp8_blocks_case(M, 1024, 1152, X.EPI_BIAS_GELU_TANH_FP8, seed=3, device=dev)
    assert _tiles(M, 1024, 128) > 2 * _sms()
    codes, scales = case.run(osb)
    torch.cuda.synchronize()
    want_codes, want_scales = X.fp8_gelu_expected(case.expected)
    X.assert_bits(str(case) + " scales", scales, want_scales)
    X.assert_bits(str(case) + " codes", codes, want_codes)


@pytest.mark.parametrize("D", [64, 72, 128])
def test_head_tiles_many_tiles(D):
    """q / k / v head tiles (bias, no norm or RoPE: one rounding of an exact value) of 200-token sequences, so row
    tiles straddle sequences."""
    import osb200 as osb

    dev = _dev()
    L, H, K = 200, 4, 1152
    rows, C = 61 * L, 4 * D
    assert _tiles(rows, 3 * C, 2 * D) > 2 * _sms()
    g = torch.Generator(device=dev).manual_seed(D)
    a = X._bf16_operand(rows, K, g)
    w = X._bf16_operand(3 * C, K, g)
    bias = X._quarters((3 * C,), g)
    want = (a.double() @ w.double().t() + bias.double()).to(torch.bfloat16)
    tiles = osb.HeadTiles(rows, osb.tile_map(0, L), 3, H, D, dev)
    osb.gemm_head_tiles(a, w, bias, tiles, nkinds=3)
    torch.cuda.synchronize()
    for kind in range(3):
        X.assert_bits(f"head tiles D={D} kind {kind}", read_tiles(tiles, kind), want[:, kind * C:(kind + 1) * C])


def test_gated_gelu_many_tiles():
    """T5's gated GELU (text mode): wi_0 pre-activations in [1024, 7168] (gelu_tanh is the identity there), wi_1 integer,
    so gelu(v0) * v1 is exact in fp32 and rounds once."""
    import osb200 as osb

    dev = _dev()
    K, d_ff = 320, 1096
    assert _tiles(M, 2 * d_ff, 256) > 2 * _sms()
    g = torch.Generator(device=dev).manual_seed(5)
    a = X._bf16_operand(M, K, g, (0, 0), zeros=False)
    wi0 = X._bf16_operand(d_ff, K, g, (0, 0), zeros=False)
    wi1 = X._bf16_operand(d_ff, K, g, (0, 0))
    bias = torch.stack((torch.full((d_ff,), X.GELU_BIAS), torch.zeros(d_ff)), 1).reshape(-1).to(torch.bfloat16).to(dev)
    got = osb.gemm(a, osb.interleave_gated(wi0, wi1), bias, epilogue=osb.EPI_GATED_GELU)
    torch.cuda.synchronize()
    v0 = a.double() @ wi0.double().t() + X.GELU_BIAS
    v1 = a.double() @ wi1.double().t()
    assert float(v0.min()) >= X.GELU_FLOOR
    X.assert_bits("gated gelu", got, (v0 * v1).to(torch.bfloat16))


CONV = dict(nb=3, thw=(5, 19, 44), cin=64, cout=328)


@functools.lru_cache(maxsize=1)
def _conv_operands():
    """Exact operands (x in {0, +-1}, w in {0, +-1} x 2^e per output channel, bias and residual multiples of 2^-2) and
    the fp64 reference, shared by every block_n."""
    import torch.nn.functional as F

    dev = _dev()
    nb, (t, h, w), cin, cout = CONV["nb"], CONV["thw"], CONV["cin"], CONV["cout"]
    g = torch.Generator(device=dev).manual_seed(17)
    ints = lambda lo, hi, *s: torch.randint(lo, hi + 1, s, generator=g, device=dev).double()   # noqa: E731
    x = ints(-1, 1, nb, t + 2, h + 2, w + 2, cin)
    wt = ints(-1, 1, cout, cin, 3, 3, 3) * torch.ldexp(torch.ones(cout, 1, 1, 1, 1, device=dev, dtype=torch.float64),
                                                       ints(-2, 2, cout, 1, 1, 1, 1).long())
    bias = ints(-256, 256, cout) / 4
    res = ints(-256, 256, nb, t, h, w, cout) / 4
    ref = F.conv3d(x.permute(0, 4, 1, 2, 3).cpu(), wt.cpu()).permute(0, 2, 3, 4, 1).to(dev) + bias + res
    assert float(ref.abs().max()) < 2.0 ** 20   # multiples of 2^-2: exact in fp32 and in the fp64 reference
    return x, wt, bias, res, ref


@pytest.mark.parametrize("block_n", [64, 128, 192, 256])
def test_conv3d_residual_many_tiles(block_n):
    """3x3x3 convolution + bias + residual on exact operands, with boxes ragged in t, h and w and in the channels."""
    import osb200 as osb

    _dev()
    nb, (t, h, w), cout = CONV["nb"], CONV["thw"], CONV["cout"]
    Tt, Ht, Wt = X.conv_box(t, h, w)
    assert t % Tt and h % Ht and w % Wt, f"box {Tt}x{Ht}x{Wt} is not ragged in every dimension of {t}x{h}x{w}"
    assert cout % block_n and nb * -(-t // Tt) * -(-h // Ht) * -(-w // Wt) * -(-cout // block_n) > 2 * _sms()
    x, wt, bias, res, ref = _conv_operands()
    y = osb.conv3d(x.to(torch.bfloat16), osb.pack_conv_weight(wt.to(torch.bfloat16), 64, False), bias.to(torch.bfloat16),
                   out_thw=(t, h, w), residual=res.to(torch.bfloat16), block_n=block_n)
    torch.cuda.synchronize()
    X.assert_bits(f"conv3d {nb}x{t}x{h}x{w}x{cout} block_n {block_n}", y, ref.to(torch.bfloat16))


@pytest.mark.parametrize("first_res", [True, False])
def test_residual_then_plain_same_stream(first_res):
    """A gate + residual GEMM and a bias-only GEMM back to back in one stream, no synchronisation between them, each
    with several tiles per CTA: both results exact."""
    import osb200 as osb

    dev = _dev()
    res_case = X.gemm_case(M, N, 320, X.EPI_BIAS_GATE_RES, gate_mode="alias", block_n=192, seed=21, device=dev)
    plain_case = X.gemm_case(M, N, 1152, X.EPI_BIAS, block_n=128, seed=22, device=dev)
    order = [res_case, plain_case] if first_res else [plain_case, res_case]
    outs = [c.run(osb) for c in order]
    torch.cuda.synchronize()
    for c, got in zip(order, outs):
        X.assert_bits(str(c), got, c.expected.to(torch.bfloat16))


def test_two_calls_identical_bits():
    """Random (inexact) operands: the fp32 summation order of every tile is fixed, so two calls agree bit for bit."""
    import osb200 as osb

    dev = _dev()
    g = torch.Generator(device=dev).manual_seed(9)
    a = torch.randn(M, 1152, device=dev, generator=g).to(torch.bfloat16)
    w = (torch.randn(N, 1152, device=dev, generator=g) / 34).to(torch.bfloat16)
    bias = torch.randn(N, device=dev, generator=g).to(torch.bfloat16)
    res = torch.randn(M, N, device=dev, generator=g).to(torch.bfloat16)
    gate = torch.randn(1, N, device=dev, generator=g)
    one = osb.gemm(a, w, bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=res, gate=gate)
    two = osb.gemm(a, w, bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=res, gate=gate)
    torch.cuda.synchronize()
    assert torch.equal(one.view(torch.int16), two.view(torch.int16))


@pytest.mark.parametrize("epi,gm", [(X.EPI_BIAS, None), (X.EPI_BIAS_GATE_RES, "alias")])
def test_fewer_tiles_than_sms(epi, gm):
    import osb200 as osb

    dev = _dev()
    case = X.gemm_case(300, 520, 1152, epi, gate_mode=gm, block_n=128, seed=4, device=dev)
    assert _tiles(300, 520, 128) < _sms()
    got = case.run(osb)
    torch.cuda.synchronize()
    X.assert_bits(str(case), got, case.expected.to(torch.bfloat16))
