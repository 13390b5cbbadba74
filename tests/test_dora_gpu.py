"""DoRA on the GPU: `osb_gemm_lora` with a per-output-channel `col_scale` (g * (x W^T + U B^T) + bias in one fp32
accumulator) against the fp32 restatement of tests/fake_osb200.py on identical bf16 operands, its bit-exactness
rules (NULL and all-ones scales), graph replay, and the MMDiT with a DoRA adapter on every Linear against the fp32 oracle
(oracle/mmdit_oracle.py) on the fp32-merged weights g * (W + s B A)."""
import pytest
import torch

from tests.fake_osb200 import gemm_lora_fp32
from tests.util import BF16_ONE_ROUNDING_REL_L2, rel_l2, report

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def osb():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import osb200

    osb200.init(0)
    return osb200


def _randn(*shape, scale=1.0, seed=0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def _operands(M, N, K, r, seed=0):
    """x, W, bias, U, s B (base product and update both ~ N(0, 1) per element) and g in [0.5, 1.5]."""
    a = _randn(M, K, seed=seed)
    w = _randn(N, K, scale=K ** -0.5, seed=seed + 1)
    bias = _randn(N, scale=0.1, seed=seed + 2)
    u = _randn(M, r, seed=seed + 3)
    b = _randn(N, r, scale=r ** -0.5, seed=seed + 4)
    g = torch.rand(N, device="cuda", generator=torch.Generator(device="cuda").manual_seed(seed + 5)) + 0.5
    return a, w, bias, u, b, g


# (M, N, K, r, block_n): ragged M, ragged N (not a multiple of the tile width), r below, at and above one 64-wide k-block
# and not a multiple of 64, every tile width
CASES = [(1, 3072, 3072, 16, 0), (3, 200, 72, 8, 64), (200, 1000, 3072, 72, 128), (777, 1032, 3072, 136, 192),
         (4096, 3072, 3072, 64, 256), (4096, 264, 3072, 24, 192), (130, 9216, 3072, 128, 0)]


@pytest.mark.parametrize("M,N,K,r,bn", CASES)
def test_gemm_lora_col_scale_bias(osb, M, N, K, r, bn):
    a, w, bias, u, b, g = _operands(M, N, K, r)
    out = osb.gemm_lora(a, w, bias, u, b, block_n=bn, col_scale=g)
    ref = gemm_lora_fp32(a, w, bias, u, b, col_scale=g)
    r_, _ = report(f"gemm_lora col_scale M={M} N={N} K={K} r={r} bn={bn}", out, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2
    # g in [0.5, 1.5]: a kernel that dropped the scale (or applied it after the bias) would be far off
    assert rel_l2(out, gemm_lora_fp32(a, w, bias, u, b)) > 0.1


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_gemm_lora_col_scale_gelu(osb, bn):
    a, w, bias, u, b, g = _operands(777, 1032, 3072, 72, seed=10)
    out = osb.gemm_lora(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GELU_TANH, block_n=bn, col_scale=g)
    ref = gemm_lora_fp32(a, w, bias, u, b, col_scale=g, epilogue=osb.EPI_BIAS_GELU_TANH)
    r_, _ = report(f"gemm_lora col_scale gelu bn={bn}", out, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("mode", ["gate_groups", "mod_index", "no_gate"])
def test_gemm_lora_col_scale_gate_residual_in_place(osb, bn, mode):
    """gate[g] * (col_scale * (x W^T + U B^T) + bias) + R with R aliasing D."""
    M, N, K, r = 600, 1152, 3072, 40
    a, w, bias, u, b, cs = _operands(M, N, K, r, seed=20)
    gate = torch.randn(4, N, device="cuda") * 0.5
    group_rows = 150
    mod_index = torch.tensor([3, 0, 2, 1], dtype=torch.int32, device="cuda") if mode == "mod_index" else None
    if mode == "no_gate":
        gate = None
    resid = _randn(M, N, seed=21)
    ref = gemm_lora_fp32(a, w, bias, u, b, col_scale=cs, epilogue=osb.EPI_BIAS_GATE_RES, residual=resid, gate=gate,
                         group_rows=group_rows, mod_index=mod_index)
    d = resid.clone()
    osb.gemm_lora(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GATE_RES, residual=d, gate=gate, group_rows=group_rows,
                  mod_index=mod_index, out=d, block_n=bn, col_scale=cs)
    r_, _ = report(f"gemm_lora col_scale gate+res {mode} bn={bn}", d, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


def test_gemm_lora_col_scale_strided_operands(osb):
    """x, U and s B as row views of wider buffers; the scale a slice of a longer (packed-group) vector."""
    M, N, K, r = 300, 512, 1024, 16
    xa = _randn(M, K + 64, seed=30)
    ua = _randn(M, 3 * r, seed=31)
    ba = _randn(2 * N, 2 * r, scale=r ** -0.5, seed=32)
    w = _randn(N, K, scale=K ** -0.5, seed=33)
    ga = torch.rand(3 * N, device="cuda") + 0.5
    a, u, b, g = xa[:, 64:], ua[:, r:2 * r], ba[N:, :r], ga[N:2 * N]
    out = osb.gemm_lora(a, w, None, u, b, col_scale=g)
    r_, _ = report("gemm_lora col_scale strided", out, gemm_lora_fp32(a, w, None, u, b, col_scale=g))
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_null_and_ones_col_scale_are_bit_identical_to_plain_lora(osb, bn):
    """x * 1.0f is exact: an all-ones scale, no scale and the call without the argument give the same bits."""
    for M, N, K, r in ((4096, 3072, 3072, 64), (3, 200, 72, 8), (777, 1032, 15360, 136)):
        a, w, bias, u, b, _ = _operands(M, N, K, r, seed=40)
        ones = torch.ones(N, device="cuda")
        resid = _randn(M, N, seed=41)
        gate = torch.randn(1, N, device="cuda")
        for kw in (dict(), dict(epilogue=osb.EPI_BIAS_GELU_TANH), dict(epilogue=osb.EPI_BIAS_GATE_RES, residual=resid, gate=gate)):
            want = osb.gemm_lora(a, w, bias, u, b, block_n=bn, **kw)
            assert torch.equal(osb.gemm_lora(a, w, bias, u, b, block_n=bn, col_scale=None, **kw), want), (M, N, K, r, bn, kw)
            assert torch.equal(osb.gemm_lora(a, w, bias, u, b, block_n=bn, col_scale=ones, **kw), want), (M, N, K, r, bn, kw)


def test_col_scale_graph_replay_equals_eager(osb):
    M, N, K, r = 1000, 3072, 3072, 64
    a, w, bias, u, b, g = _operands(M, N, K, r, seed=50)
    eager = osb.gemm_lora(a, w, bias, u, b, col_scale=g)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        osb.gemm_lora(a, w, bias, u, b, out=out, col_scale=g)   # warm-up off the capture (descriptor cache)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    out.zero_()
    with torch.cuda.graph(graph):
        osb.gemm_lora(a, w, bias, u, b, out=out, col_scale=g)
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_col_scale_argument_errors(osb):
    a, w, bias, u, b, g = _operands(64, 64, 64, 16)
    for bad in (g.double(), g[:32], torch.stack([g, g], 1)[:, 0], g.cpu(), g.to(torch.bfloat16)):
        with pytest.raises(osb.OsbError, match="col_scale"):
            osb.gemm_lora(a, w, bias, u, b, col_scale=bad)


# ---- MMDiT with a DoRA adapter on every Linear -------------------------------------------------------------------------
def test_mmdit_with_dora_vs_fp32_oracle_on_merged_weights(tmp_path):
    """tests/test_lora_gpu.py's config, inputs and bars; the magnitudes are moved off the norms of W + s B A by up to
    +-30%, so g != 1.  The adapted model against the fp32 oracle on g * (W + s B A) must be within 1e-2 and within 1.1x
    the error of the same model without the adapter against its own fp32 oracle."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import mmdit_oracle as M
    from opensora.utils.lora import load_lora, unload_lora
    from tests.adapters import merged_state_dora, write_dora_adapter
    from tests.models import MMDIT_CFG, mmdit_ids, mmdit_model

    for fused, liger in ((True, False), (False, True)):
        m = mmdit_model(fused, liger, device="cuda")
        B, Lt, (T, H, W) = 2, 40, (3, 6, 8)
        gen = torch.Generator().manual_seed(3)
        rb = lambda *s: torch.randn(*s, generator=gen).to(torch.bfloat16)  # noqa: E731
        txt_ids, img_ids = mmdit_ids(B, Lt, T, H, W)
        inp = dict(img=rb(B, T * H * W, 64), img_ids=img_ids, txt=rb(B, Lt, 128), txt_ids=txt_ids,
                   timesteps=torch.tensor([0.3, 0.8]), y_vec=rb(B, 96), cond=rb(B, T * H * W, 68),
                   guidance=torch.tensor([4.0, 7.5]))
        cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
        finp = {k: (v.float() if v.is_floating_point() else v).cuda() for k, v in inp.items()}
        dinp = {k: v.cuda() for k, v in inp.items()}

        def oracle(W32):
            return M.model_forward(W32, cfg, finp["img"], finp["img_ids"], finp["txt"], finp["txt_ids"], finp["timesteps"],
                                   finp["y_vec"], cond=finp["cond"], guidance=finp["guidance"])

        with torch.no_grad():
            base_out = m(**dinp)
            base_err = rel_l2(base_out, oracle({k: v.float() for k, v in m.state_dict().items()}))
            path = write_dora_adapter(tmp_path / f"ad_{fused}", m, r=16, alpha=32, rel=0.1, seed=5)
            load_lora(m, str(path))
            dora_out = m(**dinp)
            ref = oracle(merged_state_dora(m))
        r, _ = report(f"MMDiT + DoRA fused_qkv={fused} liger={liger}", dora_out, ref)
        print(f"[parity] same model without the adapter vs its fp32 oracle: rel_l2={base_err:.3e}")
        assert rel_l2(dora_out, base_out) > 5 * r, "the adapter must change the output well above the error"
        assert r <= 1e-2 and r <= 1.1 * base_err, (r, base_err)
        unload_lora(m)
        with torch.no_grad():
            assert torch.equal(m(**dinp), base_out)
