"""LoRA / DoRA on the FP8 GEMM (osb_gemm_fp8_lora) on the GPU: the kernel against the arithmetic of its CPU stand-in
(tests/fake_osb200.py) for every epilogue, block_n, per-row and block-scaled A, ranks of one and two tail
k-blocks and a zero-padded tail, M off the tile grid, strided U / B and gate + residual in place; exact operands (bit
for bit); NULL against all-ones col_scale; CUDA-graph replay; argument errors; and MMDiT with an adapter on every block
Linear against the fp32 oracle on the merged weights g (W + s B A), with the FP8-emulation reference as the yardstick."""
import pytest
import torch
import torch.nn.functional as F

from tests import fake_osb200 as F_
from tests import mmdit_fp8_attn_ref as AR
from tests import mmdit_fp8_lora_ref as LR
from tests import mmdit_fp8_proj_ref as PR
from tests.adapters import merged_state_dora, write_adapter, write_dora_adapter
from tests.models import MMDIT_CFG, MMDIT_WIDE, mmdit_inputs, mmdit_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu

GATE_RES, GELU, BIAS = 2, 1, 0
GELU_FP8 = F_.EPI_BIAS_GELU_TANH_FP8


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")


def _operands(M, N, K, r, seed, block_a=True, ldu=None, ldb=None):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g) * torch.logspace(-1, 1, K // 128).repeat_interleave(128)
    w = torch.randn(N, K, generator=g) / K ** 0.5
    a8, sa = F_.quant_blocks(a, 128 if block_a else K)
    w8, sw = F_.quant_blocks(w, K)
    ub = torch.zeros(M, ldu or r)
    ub[:, :r] = torch.randn(M, r, generator=g)
    bb = torch.zeros(N, ldb or r)
    bb[:, :r] = 0.3 * torch.randn(N, r, generator=g) / r ** 0.5
    u, b = ub.to(torch.bfloat16).cuda()[:, :r], bb.to(torch.bfloat16).cuda()[:, :r]
    sa = sa.cuda() if block_a else sa.view(-1).cuda()
    return g, a8.cuda(), sa, w8.cuda(), sw.view(-1).cuda(), u, b


def _reference(a8, sa, w8, sw, u, b, bias, col_scale, epilogue, res, gate, group_rows):
    """The stand-in's arithmetic in fp64, up to (not including) the rounding."""
    acc = F_.gemm_fp8_lora_acc(a8, sa, w8, sw, u, b, col_scale, torch.float64)
    if bias is not None:
        acc = acc + bias.double()
    if epilogue in (GELU, GELU_FP8):
        return F.gelu(acc, approximate="tanh")
    if epilogue == GATE_RES:
        rows = torch.arange(acc.shape[0], device=acc.device) // group_rows
        acc = acc * gate.double()[rows] + res.double()
    return acc


@pytest.mark.parametrize("M,N,K,r,block_n,epilogue,block_a", [
    (1000, 768, 512, 8, 128, BIAS, True), (300, 512, 384, 16, 64, GELU, False), (777, 384, 1024, 64, 64, GATE_RES, True),
    (1000, 1024, 768, 72, 128, GELU_FP8, True), (129, 256, 256, 128, 128, GELU_FP8, False),
    (4000, 640, 1280, 128, 0, GATE_RES, False), (513, 3072, 3072, 64, 0, BIAS, True)])
@pytest.mark.parametrize("dora", [False, True])
def test_kernel_against_the_stand_in(M, N, K, r, block_n, epilogue, block_a, dora):
    import osb200

    g, a8, sa, w8, sw, u, b = _operands(M, N, K, r, M + N + r, block_a, ldu=r + 24, ldb=r + 8)
    bias = (0.1 * torch.randn(N, generator=g)).to(torch.bfloat16).cuda()
    cs = (0.5 + torch.rand(N, generator=g)).cuda() if dora else None
    gate = torch.randn(4, N, generator=g).cuda()
    x = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    group = -(-M // 4)
    want = _reference(a8, sa, w8, sw, u, b, bias, cs, epilogue, x, gate, group)
    kw = dict(epilogue=epilogue, block_n=block_n, col_scale=cs)
    if epilogue == GATE_RES:   # in place: out aliases the residual
        before = x.clone()
        out = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, residual=x, gate=gate, group_rows=group, out=x, **kw)
        assert out.data_ptr() == x.data_ptr()
        want = _reference(a8, sa, w8, sw, u, b, bias, cs, epilogue, before, gate, group)
    elif epilogue == GELU_FP8:
        codes = torch.zeros(M, N + 256, dtype=torch.float8_e4m3fn, device="cuda")
        scales = torch.zeros(M, N // 128 + 2, device="cuda")
        osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, out=codes[:, 128:128 + N], out_scale=scales[:, 1:1 + N // 128], **kw)
        torch.cuda.synchronize()
        c, s = codes[:, 128:128 + N].float(), scales[:, 1:1 + N // 128]
        deq = (c.view(M, N // 128, 128) * s[..., None]).view(M, N)
        q, sq = F_.quant_blocks(want.float())
        err = rel_l2(deq, want.float())
        print(f"[fp8 lora gelu fp8] M={M} N={N} K={K} r={r}: rel-L2 {err:.3e}, code mismatches "
              f"{float((c != q.float()).float().mean()):.2e}")
        assert torch.allclose(s, sq, rtol=2e-3, atol=0) and err < 0.04
        # a code differs from the fp64 reference's only where the GEMM's own error (FP8 tensor-core partial sums, about
        # 2e-3 of the block's amax, i.e. of 448 code units) moves the value: by one e4m3 step (2^-3 relative, 2^-9
        # among the subnormals) plus that error
        assert (c != q.float()).float().mean() < 2e-2
        assert torch.all((c - q.float()).abs() <= 2 ** -3 * q.float().abs() + 2 ** -9 + 448 * 4e-3)
        assert not codes[:, :128].view(torch.uint8).any() and not codes[:, 128 + N:].view(torch.uint8).any()
        return
    else:
        out = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, **kw)
    torch.cuda.synchronize()
    # the bar of the FP8 block GEMM's own test (tests/test_mmdit_fp8_gpu.py): the FP8 tensor core's partial sums keep
    # fewer mantissa bits than fp32; the adapter's update is far larger than that
    err = rel_l2(out, want)
    upd = rel_l2(_reference(a8, sa, w8, sw, u, 0 * b, bias, cs, epilogue, before if epilogue == GATE_RES else x, gate,
                            group), want)
    print(f"[fp8 lora] M={M} N={N} K={K} r={r} block_n={block_n} epi={epilogue} block_a={block_a} dora={dora}: "
          f"rel-L2 {err:.2e} (the update alone moves the output by {upd:.2e})")
    assert err <= 2e-3 and upd > 20 * err


def test_exact_operands_bit_for_bit():
    """Codes in {-1, 0, 1}, power-of-two scales, integer U and B times powers of two, integer bias: every product and
    partial sum is exact in e4m3, bf16 and fp32, so any summation order gives the exact bits."""
    import osb200

    g = torch.Generator().manual_seed(1)
    M, N, K, r = 300, 384, 512, 72
    p2 = lambda *s: 2.0 ** torch.randint(-3, 4, s, generator=g).float()   # noqa: E731
    a8 = torch.randint(-1, 2, (M, K), generator=g).float().to(torch.float8_e4m3fn).cuda()
    w8 = torch.randint(-1, 2, (N, K), generator=g).float().to(torch.float8_e4m3fn).cuda()
    sa, sw = p2(M, K // 128).cuda(), p2(N).cuda()
    u = torch.randint(-4, 5, (M, r), generator=g).to(torch.bfloat16).cuda()
    b = (torch.randint(-4, 5, (N, r), generator=g).float() * p2(N, 1)).to(torch.bfloat16).cuda()
    bias = torch.randint(-8, 9, (N,), generator=g).to(torch.bfloat16).cuda()
    cs = p2(N).cuda()
    for block_n in (64, 128):
        out = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, block_n=block_n, col_scale=cs)
        want = _reference(a8, sa, w8, sw, u, b, bias, cs, BIAS, None, None, 1)
        assert torch.equal(out, want.to(torch.bfloat16))


def test_null_col_scale_equals_all_ones_and_graph_replay():
    import osb200

    g, a8, sa, w8, sw, u, b = _operands(1000, 512, 768, 64, 3)
    bias = (0.1 * torch.randn(512, generator=g)).to(torch.bfloat16).cuda()
    ones = torch.ones(512, device="cuda")
    for epi in (BIAS, GELU):
        assert torch.equal(osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, epilogue=epi),
                           osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, epilogue=epi, col_scale=ones))
    c1, s1 = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, epilogue=GELU_FP8)
    c2, s2 = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, epilogue=GELU_FP8, col_scale=ones)
    assert torch.equal(c1.view(torch.uint8), c2.view(torch.uint8)) and torch.equal(s1, s2)
    eager = osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, col_scale=ones)
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, col_scale=ones, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, bias, u, b, col_scale=ones, out=out)
    out.zero_()
    graph.replay()
    torch.cuda.synchronize()
    assert torch.equal(out, eager)


def test_argument_errors():
    import osb200

    g, a8, sa, w8, sw, u, b = _operands(256, 256, 256, 16, 5)
    with pytest.raises(osb200.OsbError, match="rank r must be a positive multiple of 8"):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u[:, :12], b[:, :12])
    with pytest.raises(osb200.OsbError, match="u must be"):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u[:100], b)
    with pytest.raises(osb200.OsbError, match="col_scale must be"):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u, b, col_scale=torch.ones(255, device="cuda"))
    with pytest.raises(osb200.OsbError, match="U and B must be 16-byte aligned"):
        big = torch.zeros(256, 40, dtype=torch.bfloat16, device="cuda")
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, big[:, 4:20], b)
    with pytest.raises(osb200.OsbError, match="col_scale must be 8-byte aligned"):
        cs = torch.ones(258, device="cuda")
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u, b, col_scale=cs[1:257])
    with pytest.raises(osb200.OsbError, match="unsupported block_n"):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u, b, block_n=192)
    with pytest.raises(osb200.OsbError, match="FP8 GELU epilogue needs block_n 128"):
        osb200.gemm_fp8_lora(a8, sa, w8, sw, None, u, b, epilogue=GELU_FP8, block_n=64)
    assert "osb_gemm_fp8_lora" in osb200.EXPORTS


# ---- the model ---------------------------------------------------------------------------------------------------------
def _adapted_case(m, cfg, inp, tmp_path, dora, attn):
    from oracle import mmdit_oracle as M
    from opensora.utils.lora import load_lora

    targets = m.fp8_mlp_linears() + m.fp8_proj_linears()
    path = str(tmp_path / "a")
    kw = dict(r=64, alpha=64, rel=0.3, seed=9, targets=targets)
    load_lora(m, write_dora_adapter(path, m, **kw) if dora else write_adapter(path, m, **kw))
    m.enable_fp8(projections=True, lora=True)
    if attn:
        m.enable_fp8_attention()
    with torch.no_grad():
        out = m(**inp)
    W32 = merged_state_dora(m)
    Wb = LR.emulation_state(m)
    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    args = lambda d, dt: (d["img"], d["img_ids"], d["txt"], d["txt_ids"], d["timesteps"].to(dt), d["y_vec"])  # noqa: E731
    ref = M.model_forward(W32, cfg, *args(f, torch.float32), cond=f["cond"], guidance=f["guidance"])
    with PR.fp8_projections(), (AR.fp8_attention() if attn else torch.no_grad()), LR.fp8_lora(m):
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    return out, emu, ref


@pytest.mark.parametrize("fused,liger,dora,attn", [(True, False, False, False), (False, True, True, True)])
def test_small_mmdit_fp8_lora_against_the_oracle(tmp_path, fused, liger, dora, attn):
    m = mmdit_model(fused, liger).cuda().to(torch.bfloat16)
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    inp = {k: v.cuda() for k, v in mmdit_inputs(2, 40, (3, 6, 8), guidance=[4.0, 7.5]).items()}
    out, emu, ref = _adapted_case(m, cfg, inp, tmp_path, dora, attn)
    r, _ = report(f"MMDiT C=256 FP8 + {'DoRA' if dora else 'LoRA'} fused={fused} liger={liger} attn={attn}", out, ref)
    r_emu = rel_l2(emu, ref)
    print(f"[mmdit fp8 lora] C=256: emulation rel_l2={r_emu:.3e}, ratio {r / r_emu:.3f}")
    # With these inputs the emulation reference itself is far from the fp32 oracle at this width (rel-L2 3.5e-2 on one
    # H100, against 6.7e-3 for the CPU test's inputs), so it is no bar here: the product is held to 1e-2, above the
    # FP8 path's own error at C = 256 (5.7e-3 to 5.8e-3 on the CPU stand-in and on the H100).
    assert r <= 1.1 * r_emu and r < 1e-2, (r, r_emu)


def test_full_width_mmdit_fp8_lora_against_the_oracle(tmp_path):
    """C = 3072 (24 x 128 heads), 2 + 2 blocks, 1 x (256 text + 2304 image) tokens, DoRA r = 64 on every block Linear,
    FP8 projections and attention."""
    m = mmdit_model(False, True, device="cuda", **MMDIT_WIDE)
    cfg = dict(MMDIT_CFG, **MMDIT_WIDE, fused_qkv=False, use_liger_rope=True)
    inp = {k: v.cuda() for k, v in mmdit_inputs(1, 256, (1, 48, 48)).items()}
    out, emu, ref = _adapted_case(m, cfg, inp, tmp_path, True, True)
    r, _ = report("MMDiT C=3072 2+2 blocks L=2560 FP8 + DoRA r=64", out, ref)
    r_emu = rel_l2(emu, ref)
    print(f"[mmdit fp8 lora] C=3072: emulation rel_l2={r_emu:.3e}, ratio {r / r_emu:.3f}")
    assert torch.isfinite(out).all() and r <= 1.1 * r_emu, (r, r_emu)
