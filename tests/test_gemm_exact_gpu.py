"""The GEMM kernels bit for bit: `gemm`, `gemm_lora` (with and without DoRA's col_scale), `gemm_fp8` and
`gemm_fp8_blocks` (including the FP8-emitting GELU epilogue) on operands whose arithmetic is exact (tests/exact_gemm.py),
one launch per case, against the fp64 reference rounded once; plus the e4m3 quantizers on rounding ties and signed zeros.

The first two tests calibrate the two hardware properties the exact cases rest on, each on one 64 x 64 tile: that the
FP8 tensor core keeps an integer k-block partial of magnitude up to 256 exact, and that tanh.approx.f32 saturates to
exactly 1.0 (so gelu_tanh is the identity for pre-activations >= 1024)."""
import pytest
import torch

from tests import exact_gemm as X

pytestmark = pytest.mark.gpu

E4M3 = torch.float8_e4m3fn


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def test_calibration_fp8_partial_256():
    """Hardware property: the FP8 wgmma sums one 128-element k-block of integer products exactly up to |256|.  Column n
    of the tile sums 128 - n products of 2 and n products of 1: partial 256 - n, bias -256, so out = -n exactly."""
    import osb200 as osb

    dev = _dev()
    a8 = torch.ones(64, 128, device=dev).to(E4M3)
    n = torch.arange(64, device=dev)
    w8 = torch.where(torch.arange(128, device=dev)[None] >= n[:, None], 2.0, 1.0).to(E4M3)
    ones = torch.ones(64, device=dev)
    bias = torch.full((64,), -256.0, device=dev).to(torch.bfloat16)
    got = osb.gemm_fp8(a8, ones, w8, ones, bias, block_n=64)
    torch.cuda.synchronize()
    want = (-n.double()).expand(64, 64).to(torch.bfloat16)
    msg = X.first_mismatch(got, want)
    print(f"[exact] calibration: FP8 k-block partial up to 256 {'exact' if msg is None else 'NOT exact: ' + msg}")
    assert msg is None, f"hardware property: the FP8 tensor core did not sum integer k-block partials <= 256 exactly: {msg}"


def test_calibration_gelu_saturation():
    """Hardware property: tanh.approx.f32 returns exactly 1.0 once gelu's argument is huge, so gelu_tanh(v) = v for v in
    [1024, 7168].  Every column's v is a bf16 rounding tie (half round up, half down under round-to-nearest-even), so a
    tanh even one ulp below 1.0 moves some column to the neighbouring bf16 value."""
    import osb200 as osb

    dev = _dev()
    K = 3072
    ulp = lambda v: 2.0 ** (int(v).bit_length() - 8)  # noqa: E731  bf16 ulp of an integer v >= 128
    vs = []
    for i in range(64):       # 64 tie values spread over [1024, 7168]
        v = 1024 + (7168 - 1024 - 64) * i // 63
        v = v - v % int(ulp(v)) + int(ulp(v)) // 2
        vs.append(v)
    v = torch.tensor(vs, dtype=torch.float64)
    j = ((7168 - v) / 2).long()      # w row n: first j_n entries -1, the rest +1, so a . w = K - 2 j_n = v - 4096
    w = torch.where(torch.arange(K)[None] < j[:, None], -1.0, 1.0).to(torch.bfloat16).to(dev)
    a = torch.ones(64, K, dtype=torch.bfloat16, device=dev)
    bias = torch.full((64,), X.GELU_BIAS, dtype=torch.bfloat16, device=dev)
    got = osb.gemm(a, w, bias, epilogue=osb.EPI_BIAS_GELU_TANH, block_n=64)
    torch.cuda.synchronize()
    want = v.to(dev).expand(64, 64).to(torch.bfloat16)
    msg = X.first_mismatch(got, want)
    print(f"[exact] calibration: tanh.approx.f32 saturation {'exact (gelu_tanh(v) = v)' if msg is None else 'NOT exact: ' + msg}")
    assert msg is None, f"hardware property: tanh.approx.f32 did not saturate to exactly 1.0 (gelu_tanh(v) != v): {msg}"


CASES = X.matrix()


@pytest.mark.parametrize("idx", range(len(CASES)), ids=[c[0] for c in CASES])
def test_gemm_exact(idx):
    import osb200 as osb

    dev = _dev()
    name, builder, args, kw = CASES[idx]
    case = builder(*args, seed=idx, device=dev, **kw)
    l0 = osb.launch_count()
    got = case.run(osb)
    torch.cuda.synchronize()
    assert osb.launch_count() == l0 + 1, "one launch per call"
    if case.epilogue == X.EPI_BIAS_GELU_TANH_FP8:
        codes, scales = got
        want_codes, want_scales = X.fp8_gelu_expected(case.expected)
        msg = X.first_mismatch(scales, want_scales) or X.first_mismatch(codes, want_codes)
        outside = case.out_buf.clone()
        outside[:, 128:128 + case.N] = 0x5A
        sc = case.scale_buf.clone()
        sc[:, 1:1 + case.N // 128] = -7.0
        assert bool((outside == 0x5A).all()) and bool((sc == -7.0).all()), f"{case}: wrote outside the output slices"
    else:
        if case.out is not None:
            assert got.data_ptr() == case.out.data_ptr()
        msg = X.first_mismatch(got, case.expected.to(torch.bfloat16))
    print(f"[exact] {case}: {'bit-identical' if msg is None else msg}")
    assert msg is None, f"{case}: {msg}"


# ---- quantizers on ties and signed zeros ------------------------------------------------------------------------------
@pytest.mark.parametrize("which", ["rows", "blocks128", "blocksK"])
def test_quantizer_edges(which):
    import osb200 as osb

    dev = _dev()
    x = X.quant_edge_rows()
    K = x.shape[1]
    if which == "rows":
        q, s = osb.quant_rows_fp8(x.to(dev))
        wq, ws = X.quant_expected(x, K)
        ws = ws[:, 0]
    else:
        block = 128 if which == "blocks128" else K
        q, s = osb.quant_blocks_fp8(x.to(dev), block=block)
        wq, ws = X.quant_expected(x, block)
    torch.cuda.synchronize()
    msg = X.first_mismatch(s.cpu(), ws, signed_zero=True) or X.first_mismatch(q.cpu(), wq, signed_zero=True)
    print(f"[exact] quantizer {which}: {'bit-identical' if msg is None else msg}")
    assert msg is None, f"quantizer {which}: {msg}"
