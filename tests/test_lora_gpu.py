"""LoRA on the GPU: `osb_gemm_lora` (base GEMM + unmerged low-rank update in one fp32 accumulator) against the fp32
restatement of tests/fake_osb200.py on identical bf16 operands, and the MMDiT with an adapter on every Linear against the
fp32 oracle (oracle/mmdit_oracle.py) on the fp32-merged weights W + s B A."""
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
    """x, W, bias, U, s B with the base product and the update of the same size (both ~ N(0, 1) per element)."""
    a = _randn(M, K, seed=seed)
    w = _randn(N, K, scale=K ** -0.5, seed=seed + 1)
    bias = _randn(N, scale=0.1, seed=seed + 2)
    u = _randn(M, r, seed=seed + 3)
    b = _randn(N, r, scale=r ** -0.5, seed=seed + 4)
    return a, w, bias, u, b


# (M, N, K, r, block_n): every M of the issue's list, ragged N (not a multiple of the tile width), K with a ragged last
# k-block (72) up to linear2's 15360, ranks below, at and above one 64-wide k-block, and every tile width
CASES = [
    (1, 3072, 3072, 16, 0), (3, 200, 72, 8, 0), (200, 1000, 3072, 72, 0), (4096, 3072, 3072, 64, 0),
    (4096, 9216, 3072, 128, 256), (200, 12288, 3072, 256, 192), (4096, 3072, 15360, 16, 128), (3, 3072, 15360, 128, 64),
    (200, 200, 72, 256, 128), (4096, 1000, 72, 8, 64), (1, 72, 3072, 72, 256), (4096, 264, 3072, 16, 192),
]


@pytest.mark.parametrize("M,N,K,r,bn", CASES)
def test_gemm_lora_bias(osb, M, N, K, r, bn):
    a, w, bias, u, b = _operands(M, N, K, r)
    out = osb.gemm_lora(a, w, bias, u, b, block_n=bn)
    ref = gemm_lora_fp32(a, w, bias, u, b)
    r_, _ = report(f"gemm_lora M={M} N={N} K={K} r={r} bn={bn}", out, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2
    # the update is half of the signal: a kernel that dropped it would be off by ~70%
    assert rel_l2(out, ref - u.float() @ b.float().t()) > 0.3


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("r", [8, 72])
def test_gemm_lora_gelu(osb, bn, r):
    a, w, bias, u, b = _operands(777, 1032, 3072, r, seed=10)
    out = osb.gemm_lora(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GELU_TANH, block_n=bn)
    ref = gemm_lora_fp32(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GELU_TANH)
    r_, _ = report(f"gemm_lora gelu bn={bn} r={r}", out, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
@pytest.mark.parametrize("mode", ["gate_groups", "mod_index", "no_gate"])
def test_gemm_lora_gate_residual_in_place(osb, bn, mode):
    """gate[g] * (x W^T + U B^T + bias) + R with R aliasing D; g by group_rows, or through mod_index."""
    M, N, K, r = 600, 1152, 3072, 128
    a, w, bias, u, b = _operands(M, N, K, r, seed=20)
    gate = torch.randn(4, N, device="cuda") * 0.5
    group_rows = 150
    mod_index = torch.tensor([3, 0, 2, 1], dtype=torch.int32, device="cuda") if mode == "mod_index" else None
    if mode == "no_gate":
        gate = None
    resid = _randn(M, N, seed=21)
    ref = gemm_lora_fp32(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GATE_RES, residual=resid, gate=gate,
                         group_rows=group_rows, mod_index=mod_index)
    d = resid.clone()
    osb.gemm_lora(a, w, bias, u, b, epilogue=osb.EPI_BIAS_GATE_RES, residual=d, gate=gate, group_rows=group_rows,
                  mod_index=mod_index, out=d, block_n=bn)
    r_, _ = report(f"gemm_lora gate+res {mode} bn={bn}", d, ref)
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


def test_gemm_lora_strided_operands(osb):
    """x, U and s B as row views of wider buffers (U of a shared down projection, B a row block of a packed one)."""
    M, N, K, r = 300, 512, 1024, 16
    xa = _randn(M, K + 64, seed=30)
    ua = _randn(M, 3 * r, seed=31)
    ba = _randn(2 * N, 2 * r, scale=r ** -0.5, seed=32)
    w = _randn(N, K, scale=K ** -0.5, seed=33)
    a, u, b = xa[:, 64:], ua[:, r:2 * r], ba[N:, :r]
    out = osb.gemm_lora(a, w, None, u, b)
    r_, _ = report("gemm_lora strided", out, gemm_lora_fp32(a, w, None, u, b))
    assert r_ <= BF16_ONE_ROUNDING_REL_L2


@pytest.mark.parametrize("bn", [64, 128, 192, 256])
def test_zero_update_is_bit_identical_to_gemm(osb, bn):
    """B = 0: the extra k-blocks add exact zeros, so the base K loop must give osb_gemm_bf16's bits."""
    for M, N, K, r in ((4096, 3072, 3072, 64), (3, 200, 72, 8), (777, 1032, 15360, 256)):
        a, w, bias, u, _ = _operands(M, N, K, r, seed=40)
        zero = torch.zeros(N, r, dtype=torch.bfloat16, device="cuda")
        resid = _randn(M, N, seed=41)
        gate = torch.randn(1, N, device="cuda")
        for kw in (dict(), dict(epilogue=osb.EPI_BIAS_GELU_TANH), dict(epilogue=osb.EPI_BIAS_GATE_RES, residual=resid, gate=gate)):
            want = osb.gemm(a, w, bias, block_n=bn, **kw)
            got = osb.gemm_lora(a, w, bias, u, zero, block_n=bn, **kw)
            assert torch.equal(got, want), (M, N, K, r, bn, kw)


def test_graph_replay_equals_eager(osb):
    M, N, K, r = 1000, 3072, 3072, 64
    a, w, bias, u, b = _operands(M, N, K, r, seed=50)
    eager = osb.gemm_lora(a, w, bias, u, b)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        osb.gemm_lora(a, w, bias, u, b, out=out)   # warm-up off the capture (descriptor cache)
    torch.cuda.current_stream().wait_stream(s)
    g = torch.cuda.CUDAGraph()
    out.zero_()
    with torch.cuda.graph(g):
        osb.gemm_lora(a, w, bias, u, b, out=out)
    g.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_gemm_lora_argument_errors(osb):
    a, w, bias, u, b = _operands(64, 64, 64, 16)
    with pytest.raises(osb.OsbError, match="multiple of 8"):
        osb.gemm_lora(a, w, bias, u[:, :12], b[:, :12])
    with pytest.raises(osb.OsbError):
        osb.gemm_lora(a, w, bias, u, b[:, :8])


# ---- MMDiT with an adapter on every Linear ----------------------------------------------------------------------------
def test_mmdit_with_adapter_vs_fp32_oracle_on_merged_weights(tmp_path):
    """tests/test_mmdit_gpu.py's config and inputs; adapter updates about 10% of |W| per Linear.  The adapted model against
    the fp32 oracle on W + s B A must be within 1e-2 and within 1.1x the error of the same model without the adapter
    against its own fp32 oracle."""
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from oracle import mmdit_oracle as M
    from opensora.utils.lora import load_lora, unload_lora
    from tests.adapters import merged_state, write_adapter
    from tests.models import MMDIT_CFG, mmdit_ids, mmdit_model

    results = {}
    for fused, liger in ((True, False), (False, True)):
        m = mmdit_model(fused, liger, device="cuda")
        B, Lt, (T, H, W) = 2, 40, (3, 6, 8)
        g = torch.Generator().manual_seed(3)
        rb = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
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
            path = write_adapter(tmp_path / f"ad_{fused}", m, r=16, alpha=32, rel=0.1, seed=5)
            load_lora(m, str(path))
            lora_out = m(**dinp)
            ref = oracle(merged_state(m))
        r, _ = report(f"MMDiT + LoRA fused_qkv={fused} liger={liger}", lora_out, ref)
        print(f"[parity] same model without the adapter vs its fp32 oracle: rel_l2={base_err:.3e}")
        assert rel_l2(lora_out, base_out) > 5 * r, "the adapter must change the output well above the error"
        results[(fused, liger)] = (r, base_err)
        assert r <= 1e-2 and r <= 1.1 * base_err, (r, base_err)
        unload_lora(m)
        with torch.no_grad():
            assert torch.equal(m(**dinp), base_out)
