"""The block-scaled FP8 (e4m3) MLP path of MMDiT on the H100: `osb_gemm_fp8_blocks` against an fp32 matmul of the
dequantized operands (K = 3072, 12 288, 15 360, every epilogue, ragged M, partial last column tiles), its per-row mode
against `osb_gemm_fp8`, the FP8-emitting GELU epilogue, `osb_quant_blocks_fp8` against the CPU stand-in, and MMDiTModel
with FP8 MLPs against the fp32 oracle (yardstick: the FP8-emulation reference of tests/mmdit_fp8_ref.py, measured in the
same test) at the small config of tests/test_mmdit_gpu.py and at full width (C = 3072, 24 x 128 heads)."""
import pytest
import torch
import torch.nn.functional as F

from tests import fake_osb200 as F_
from tests import mmdit_fp8_ref as MR
from tests.models import MMDIT_CFG, MMDIT_WIDE, mmdit_inputs, mmdit_model
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _operands(M, N, K, seed):
    g = torch.Generator().manual_seed(seed)
    a = torch.randn(M, K, generator=g) * torch.logspace(-2, 1, K // 128).repeat_interleave(128)
    a = a * torch.logspace(-1, 1, M)[:, None]
    w = torch.randn(N, K, generator=g) / K ** 0.5
    a8, sa = F_.quant_blocks(a)
    w8, sw = F_.quant_blocks(w, K)
    return g, a8.cuda(), sa.cuda(), w8.cuda(), sw.view(-1).cuda()


def _deq(a8, sa):
    M, K = a8.shape
    return (a8.float().view(M, K // 128, 128) * sa[..., None]).view(M, K)


@pytest.mark.parametrize("M,N,K,block_n", [(2048, 3072, 12288, 0), (1500, 3072, 15360, 0), (2000, 12288, 3072, 0),
                                           (333, 520, 3072, 128), (77, 520, 15360, 64), (129, 384, 12288, 64),
                                           (50, 40, 3072, 0)])
@pytest.mark.parametrize("epilogue", [0, 1, 2])
def test_block_gemm_against_dequantized_fp32(M, N, K, block_n, epilogue):
    import osb200

    g, a8, sa, w8, sw = _operands(M, N, K, M + N + K + epilogue)
    bias = (0.1 * torch.randn(N, generator=g)).to(torch.bfloat16).cuda()
    res = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    gate = torch.randn(6, N, generator=g).cuda()
    group_rows = -(-M // 3)
    mod_index = torch.tensor([4, 1, 5], dtype=torch.int32).cuda()
    kw = dict(residual=res, gate=gate, group_rows=group_rows, mod_index=mod_index) if epilogue == 2 else {}
    # a_scale as a column view of a wider buffer (row stride > K / 128)
    sa_view = torch.zeros(M, K // 128 + 3, device="cuda")[:, 1:1 + K // 128]
    sa_view.copy_(sa)
    out = osb200.gemm_fp8_blocks(a8, sa_view, w8, sw, bias, epilogue=epilogue, block_n=block_n, **kw)
    ref = _deq(a8, sa) @ (w8.float() * sw[:, None]).t() + bias.float()
    if epilogue == 1:
        ref = F.gelu(ref, approximate="tanh")
    elif epilogue == 2:
        gi = mod_index.long()[torch.arange(M, device="cuda") // group_rows]
        ref = ref * gate[gi] + res.float()
    torch.cuda.synchronize()
    r = rel_l2(out, ref)
    print(f"[gemm_fp8_blocks] M{M} N{N} K{K} bn{block_n} epi{epilogue}: rel_l2 {r:.2e}")
    assert r <= 2e-3


@pytest.mark.parametrize("epilogue", [0, 1, 2])
def test_per_row_mode_is_gemm_fp8(epilogue):
    """Per-row scales through osb_gemm_fp8_blocks give the bits of osb_gemm_fp8."""
    import osb200

    M, N, K = 1000, 640, 3072
    g = torch.Generator().manual_seed(9)
    a8, sa = (t.cuda() for t in F_._quant(torch.randn(M, K, generator=g)))
    w8, sw = (t.cuda() for t in F_._quant(torch.randn(N, K, generator=g) / K ** 0.5))
    bias = torch.randn(N, generator=g).to(torch.bfloat16).cuda()
    res = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    gate = torch.randn(2, N, generator=g).cuda()
    kw = dict(residual=res, gate=gate, group_rows=500) if epilogue == 2 else {}
    want = osb200.gemm_fp8(a8, sa, w8, sw, bias, epilogue=epilogue, **kw)
    got = osb200.gemm_fp8_blocks(a8, sa, w8, sw, bias, epilogue=epilogue, **kw)
    assert torch.equal(got, want)


@pytest.mark.parametrize("M,N,K,block_scaled", [(2000, 12288, 3072, False), (333, 1024, 3072, True),
                                                 (129, 384, 12288, True), (70, 128, 256, False)])
def test_gelu_fp8_epilogue(M, N, K, block_scaled):
    """Every block's scale is amax / 448 of its dequantized values and some code of each nonzero block is +-448; the
    dequantized output is the bf16-epilogue GEMM's GELU output within one e4m3 rounding plus the GEMM's own error.  The
    codes land in a column slice of a wider buffer."""
    import osb200

    g, a8, sa, w8, sw = _operands(M, N, K, M + N)
    if not block_scaled:
        sa = sa[:, 0].contiguous()   # per-row A (the fc1 input of ln_modulate_fp8)
    bias = (0.3 * torch.randn(N, generator=g)).to(torch.bfloat16).cuda()
    cat = torch.zeros(M, N + 256, dtype=E4M3, device="cuda")
    cats = torch.full((M, N // 128 + 2), -1.0, device="cuda")
    q, s = osb200.gemm_fp8_blocks(a8, sa, w8, sw, bias, epilogue=osb200.EPI_BIAS_GELU_TANH_FP8, out=cat[:, 128:128 + N],
                                  out_scale=cats[:, 1:1 + N // 128])
    bf = osb200.gemm_fp8_blocks(a8, sa, w8, sw, bias, epilogue=osb200.EPI_BIAS_GELU_TANH).float()
    sa2 = sa if block_scaled else sa[:, None].expand(M, K // 128)
    ref = F.gelu(_deq(a8, sa2) @ (w8.float() * sw[:, None]).t() + bias.float(), approximate="tanh")
    torch.cuda.synchronize()
    assert not cat[:, :128].float().any() and not cat[:, 128 + N:].float().any()
    assert (cats[:, 0] == -1).all() and (cats[:, -1] == -1).all()
    qb = q.float().view(M, N // 128, 128)
    deq = qb * s[..., None]
    amax = deq.abs().amax(-1)
    nz = amax > 0
    assert torch.allclose(s[nz], amax[nz] / 448, rtol=1e-6, atol=0) and (s[~nz] == 1).all()
    assert (qb.abs().amax(-1)[nz] == 448).all()
    deq = deq.view(M, N)
    sb = s.repeat_interleave(128, dim=1)
    # e4m3 rounding: half a step (2^-4 |v|, 2^-10 s among the subnormals); bf16 rounding of the reference output 2^-8 |v|;
    # the GEMM's own error (the per-row bf16 epilogue runs osb_gemm_fp8, which applies the row scale after the sum)
    bound = (2.0 ** -4 + 2.0 ** -8) * 1.01 * bf.abs() + 2.0 ** -10 * sb + 1e-4 * 448 * sb
    err = (deq - bf).abs()
    print(f"[gelu_fp8] M{M} N{N} K{K}: max |deq - bf16 GELU| / bound {(err / bound).max():.3f}, "
          f"rel_l2 to fp32 {rel_l2(deq, ref):.2e}")
    assert (err <= bound).all()


@pytest.mark.parametrize("rows,K,block,ld", [(26484, 3072, 128, 15360), (1000, 15360, 15360, 15360),
                                              (37, 12288, 12288, 12416), (300, 3072, 3072, 3072), (5, 256, 128, 384)])
def test_quant_blocks_fp8_matches_the_stand_in(rows, K, block, ld):
    import osb200

    g = torch.Generator().manual_seed(rows + K)
    x = (torch.randn(rows, ld, generator=g) * torch.logspace(-4, 2, rows)[:, None]).to(torch.bfloat16)
    x[1] = 0
    x[2, 5] = 3e4
    q, s = osb200.quant_blocks_fp8(x.cuda()[:, :K], block=block)
    rq, rs = F_.quant_blocks_fp8(x[:, :K], block=block)
    assert torch.equal(s.cpu(), rs)
    assert torch.equal(q.cpu().view(torch.uint8), rq.view(torch.uint8))


def _check_model(m, cfg, inp, tag):
    from oracle import mmdit_oracle as M

    plain_out = None
    with torch.no_grad():
        plain_out = m(**inp).clone()
    m.enable_fp8()
    got_x = []
    hooks = [b.register_forward_hook(lambda mod, a, out: got_x.append(
        torch.cat((out[1], out[0]), 1).float() if isinstance(out, tuple) else out.float())) for b in list(m.double_blocks) + list(m.single_blocks)]
    try:
        with torch.no_grad():
            out = m(**inp)
    finally:
        for h in hooks:
            h.remove()
    W32 = {k: v.float() for k, v in m.state_dict().items()}
    Wb = dict(m.state_dict())
    f = {k: (v.float() if v.is_floating_point() else v) for k, v in inp.items()}
    args = lambda d, dt: (d["img"], d["img_ids"], d["txt"], d["txt_ids"], d["timesteps"].to(dt), d["y_vec"])  # noqa: E731
    ref_x = []
    od, os_ = M.double_stream_block, M.single_stream_block

    def dbl(*a, **k):
        i, t = od(*a, **k)
        ref_x.append(torch.cat((t, i), 1).float())
        return i, t

    def sgl(*a, **k):
        x = os_(*a, **k)
        ref_x.append(x.float())
        return x

    M.double_stream_block, M.single_stream_block = dbl, sgl
    try:
        ref = M.model_forward(W32, cfg, *args(f, torch.float32), cond=f["cond"], guidance=f["guidance"])
    finally:
        M.double_stream_block, M.single_stream_block = od, os_
    with MR.fp8_mlps():
        emu = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    floor = M.model_forward(Wb, cfg, *args(inp, torch.bfloat16), cond=inp["cond"], guidance=inp["guidance"].to(torch.bfloat16))
    per_block = [rel_l2(g, r) for g, r in zip(got_x, ref_x)]
    r, _ = report(f"MMDiT {tag} FP8 MLPs", out, ref)
    r_emu, r_bf = rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[mmdit fp8] {tag}: FP8-emulation reference rel_l2={r_emu:.3e}, bf16 oracle rel_l2={r_bf:.3e}, "
          f"ratio {r / r_emu:.3f}")
    print(f"[mmdit fp8] {tag}: residual stream rel_l2 after block k: " +
          " ".join(f"{k}:{e:.1e}" for k, e in enumerate(per_block)))
    assert torch.isfinite(out).all() and len(per_block) == cfg["depth"] + cfg["depth_single_blocks"]
    for k in range(1, len(per_block)):
        assert per_block[k] < 3.0 * per_block[k - 1], (k, per_block[k - 1], per_block[k])
    assert r <= 1.1 * r_emu, (r, r_emu)
    m.disable_fp8()
    with torch.no_grad():
        back = m(**inp)
    assert torch.equal(back, plain_out)


@pytest.mark.parametrize("fused,liger", [(True, False), (False, True)])
def test_small_mmdit_fp8_against_the_oracle(fused, liger):
    m = mmdit_model(fused, liger, device="cuda")
    cfg = dict(MMDIT_CFG, fused_qkv=fused, use_liger_rope=liger)
    inp = {k: v.cuda() for k, v in mmdit_inputs(2, 40, (3, 6, 8), guidance=[4.0, 7.5]).items()}
    _check_model(m, cfg, inp, f"C=256 fused_qkv={fused} liger={liger}")


def test_full_width_mmdit_fp8_against_the_oracle():
    """C = 3072 (24 x 128 heads), 2 + 2 blocks, 1 x (256 text + 2304 image) tokens."""
    m = mmdit_model(False, True, device="cuda", **MMDIT_WIDE)
    cfg = dict(MMDIT_CFG, **MMDIT_WIDE, fused_qkv=False, use_liger_rope=True)
    inp = {k: v.cuda() for k, v in mmdit_inputs(1, 256, (1, 48, 48)).items()}
    _check_model(m, cfg, inp, "C=3072 2+2 blocks L=2560")
