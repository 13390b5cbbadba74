"""The FP8 (e4m3) MLP path on the H100: `osb_gemm_fp8` against an fp32 matmul of the dequantized operands, the two
quantizers against their CPU stand-in (tests/fake_osb200.py), STDiT3-XL/2 at the benchmark shape with FP8 MLPs
against the fp32 oracle (yardstick: the FP8-emulation reference of tests/fp8_ref.py, measured in the same test), graph
replay, and `disable_fp8()`."""
import pytest
import torch
import torch.nn.functional as F

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests.models import stdit3_inputs, stdit3_pair
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _q(x):
    """quantize on the CPU stand-in's rule, return device tensors (codes as e4m3, scales fp32)"""
    q, s = F_._quant(x.float().cpu())
    return q.cuda(), s.cuda()


@pytest.mark.parametrize("M,N,K,block_n", [(16384, 4608, 1152, 0), (16384, 1152, 4608, 0), (300, 256, 1152, 64),
                                           (1000, 384, 384, 128), (129, 576, 256, 64), (77, 512, 4608, 128),
                                           (600, 520, 1152, 128), (200, 520, 4608, 64), (50, 40, 256, 0)])
@pytest.mark.parametrize("epilogue", [0, 1, 2])
def test_gemm_fp8_against_dequantized_fp32(M, N, K, block_n, epilogue):
    import osb200

    g = torch.Generator().manual_seed(M + N + K + epilogue)
    a = torch.randn(M, K, generator=g) * torch.logspace(-2, 1, M)[:, None]
    w = torch.randn(N, K, generator=g) / K ** 0.5
    a8, sa = _q(a)
    w8, sw = _q(w)
    bias = (0.1 * torch.randn(N, generator=g)).to(torch.bfloat16).cuda()
    res = torch.randn(M, N, generator=g).to(torch.bfloat16).cuda()
    G = 6
    gate = torch.randn(G, N, generator=g).cuda()
    group_rows = -(-M // 3)
    mod_index = torch.tensor([4, 1, 5], dtype=torch.int32).cuda()
    kw = dict(residual=res, gate=gate, group_rows=group_rows, mod_index=mod_index) if epilogue == 2 else {}
    out = osb200.gemm_fp8(a8, sa, w8, sw, bias, epilogue=epilogue, block_n=block_n, **kw)
    ref = (a8.float() * sa[:, None]) @ (w8.float() * sw[:, None]).t() + bias.float()
    if epilogue == 1:
        ref = F.gelu(ref, approximate="tanh")
    elif epilogue == 2:
        gi = mod_index.long()[torch.arange(M, device="cuda") // group_rows]
        ref = ref * gate[gi] + res.float()
    torch.cuda.synchronize()
    r = rel_l2(out, ref)
    print(f"[gemm_fp8] M{M} N{N} K{K} bn{block_n} epi{epilogue}: rel_l2 {r:.2e}")
    assert r <= 2e-3   # summation order and one bf16 rounding (N = 520, 40: a partial last column tile)


def test_gemm_fp8_refusals():
    import osb200

    z = torch.zeros(128, 288, dtype=E4M3, device="cuda")
    s = torch.ones(128, device="cuda")
    with pytest.raises(osb200.OsbError, match="multiple of 128"):
        osb200.gemm_fp8(z, s, z, s)
    z = torch.zeros(128, 256, dtype=E4M3, device="cuda")
    with pytest.raises(osb200.OsbError, match="not built for FP8"):
        osb200.gemm_fp8(z, s, z, s, epilogue=osb200.EPI_GATED_GELU)
    with pytest.raises(osb200.OsbError, match="unsupported block_n"):
        osb200.gemm_fp8(z, s, z, s, block_n=256)


def _step(q):
    return (q.abs() * 2.0 ** -3).clamp(min=2.0 ** -9)


@pytest.mark.parametrize("rows,K,ld", [(16384, 4608, 4608), (1000, 1152, 1152), (37, 288, 320), (64, 8192, 8192)])
def test_quant_rows_fp8_matches_the_stand_in(rows, K, ld):
    import osb200

    g = torch.Generator().manual_seed(rows + K)
    x = (torch.randn(rows, ld, generator=g) * torch.logspace(-4, 2, rows)[:, None]).to(torch.bfloat16)
    x[1] = 0
    x[2, 5] = 3e4
    xs = x.cuda()[:, :K]
    q, s = osb200.quant_rows_fp8(xs)
    rq, rs = F_.quant_rows_fp8(x[:, :K])
    assert torch.equal(s.cpu(), rs)                    # amax is exact and amax / 448 is one IEEE division
    qc, rc = q.cpu().float(), rq.float()
    assert ((qc - rc).abs() <= _step(rc)).all()
    mism = (qc != rc).float().mean().item()
    print(f"[quant_rows_fp8] {rows}x{K}: codes differing {mism:.2e}")
    assert mism == 0.0


@pytest.mark.parametrize("rows,C,x_mask", [(16384, 1152, False), (2048, 1152, True), (500, 256, True), (64, 4096, False)])
def test_ln_modulate_fp8_matches_the_stand_in(rows, C, x_mask):
    import osb200

    g = torch.Generator().manual_seed(rows + C)
    x = (torch.randn(rows, C, generator=g) * 2).to(torch.bfloat16)
    x[3] = 1.5
    mod = torch.randn(4, 2, C, generator=g) * 0.5
    group_rows = -(-rows // 4) if not x_mask else -(-rows // 8)   # every group index stays inside the tables
    mod_index = torch.tensor([1, 0, 3, 2, 2, 3, 0, 1], dtype=torch.int32) if x_mask else None
    q, s = osb200.ln_modulate_fp8(x.cuda(), mod[:, 0].cuda(), mod[:, 1].cuda(), group_rows=group_rows,
                                  mod_index=None if mod_index is None else mod_index.cuda())
    rq, rs = F_.ln_modulate_fp8(x, mod[:, 0], mod[:, 1], group_rows=group_rows, mod_index=mod_index)
    sc = s.cpu()
    assert ((sc - rs).abs() <= 1e-6 * rs).all()
    qc, rc = q.cpu().float(), rq.float()
    assert ((qc - rc).abs() <= _step(rc)).all()        # fp32 statistics summed in another order: a near-tie may flip
    mism = (qc != rc).float().mean().item()
    print(f"[ln_modulate_fp8] {rows}x{C}: codes differing {mism:.2e}")
    assert mism < 1e-3


def test_xl_fp8_at_the_benchmark_shape():
    """STDiT3-XL/2, full depth, 1x4x64x32x32 (16 384 tokens), FP8 MLPs, against the fp32 oracle holding the same bf16
    weights.  Bars: the error is at most 1.1x that of the FP8-emulation reference (the oracle in bf16 with its block
    MLPs at the FP8 rounding points), and the residual stream never jumps by more than 3x between consecutive blocks."""
    prod, oracle, cfg = stdit3_pair("xl")
    prod.enable_fp8()
    inp = stdit3_inputs(cfg, 1, 64, 32, 32, lens=[260], device="cuda")
    oracle = oracle.cuda()
    ref_x, got_x = [], []
    hooks = [b.register_forward_hook(lambda m, a, out: ref_x.append(out.detach().float()))
             for pair in zip(oracle.spatial_blocks, oracle.temporal_blocks) for b in pair]
    orig = prod._block

    def traced(osb, blk, bi, xs, *a, **k):
        r = orig(osb, blk, bi, xs, *a, **k)
        got_x.append(xs.detach().float().clone())
        return r

    prod._block = traced
    try:
        with torch.no_grad():
            ref = oracle(**inp)
            out = prod(**inp)
    finally:
        prod._block = orig
        for h in hooks:
            h.remove()
    per_block = [rel_l2(g.view_as(r), r) for g, r in zip(got_x, ref_x)]
    del ref_x, got_x
    with torch.no_grad():
        ob = oracle.to(torch.bfloat16)
        floor = ob(**inp).float()
        with R.fp8_mlps(ob):
            emu = ob(**inp).float()
    r, _ = report("STDiT3-XL/2 64x32x32 FP8 MLPs", out, ref)
    r_emu, r_bf = rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[fp8] FP8-emulation reference rel_l2={r_emu:.3e}, bf16 oracle rel_l2={r_bf:.3e}, ratio {r / r_emu:.3f}")
    print("[fp8] residual stream rel_l2 after block k: " + " ".join(f"{k}:{e:.1e}" for k, e in enumerate(per_block)))
    assert torch.isfinite(out).all() and len(per_block) == 2 * cfg.depth
    for k in range(1, len(per_block)):
        assert per_block[k] < 3.0 * per_block[k - 1], (k, per_block[k - 1], per_block[k])
    assert r <= 1.1 * r_emu, (r, r_emu)


def test_enable_fp8_stays_off_when_quantization_fails():
    """fp32 weights on the GPU: the weight quantizer refuses them, and the model keeps running its bf16 MLPs."""
    import osb200

    prod = stdit3_pair("xs64")[0].float()
    with pytest.raises(osb200.OsbError):
        prod.enable_fp8()
    assert prod._fp8 is False and not any(k[0] == "fp8" for k in prod._cache)


def test_fp8_graph_replay_and_disable():
    """XS/2 at hidden 256 with an x_mask: the captured FP8 step replays to the eager bits; disable_fp8() gives the bits
    of a model that never enabled FP8."""
    prod, oracle, cfg = stdit3_pair("xs64")
    plain = stdit3_pair("xs64")[0]
    inp = stdit3_inputs(cfg, 2, 8, 16, 16, lens=[300, 21], device="cuda")
    xm = torch.ones(2, 8, dtype=torch.bool, device="cuda")
    xm[1, :3] = False
    with torch.no_grad():
        want_bf16 = plain(**inp, x_mask=xm)
        prod.enable_fp8()
        eager = prod(**inp, x_mask=xm).clone()
        ref = oracle.cuda()(**inp, x_mask=xm)
    replay = prod.capture(**inp, x_mask=xm)
    got = replay(**inp, x_mask=xm).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, eager)
    assert rel_l2(eager, ref) < 3e-2
    assert not torch.equal(eager, want_bf16)
    del replay
    prod.disable_fp8()
    with torch.no_grad():
        back = prod(**inp, x_mask=xm)
    assert torch.equal(back, want_bf16)
