"""The FP8 (e4m3) head-tile attention of STDiT3 on the H100: `osb_head_tiles_fp8` bit for bit against its CPU stand-in
(tests/fake_osb200.py) on the bf16 tiles the projection GEMM wrote, `osb_attn_tiles_fp8` against fp32 softmax
on the dequantized e4m3 tiles (bar: 1.1x the error of the P-emulation on the same operands) for every set shape of the
model, the peer-scatter routing, repeatability, STDiT3-XL/2 at the benchmark shape against the fp32 oracle (yardstick:
tests/stdit3_fp8_attn_ref.py), graph replay and `disable_fp8_attention()`."""
import types

import pytest
import torch

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests import stdit3_fp8_attn_ref as A
from tests.models import stdit3_inputs, stdit3_pair
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu
E4M3 = torch.float8_e4m3fn


@pytest.fixture(autouse=True)
def _cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _osb():
    import osb200

    osb200.init(0)
    return osb200


def bf16_tiles(t, kind):
    """fp32 [heads, tiles, 128, D] decoded from the bytes of a real HeadTiles buffer (tiles.cuh layout)."""
    TR, D = t.map.tile_rows, t.head_dim
    main = D // 64
    r = torch.arange(TR, device="cuda")[:, None]
    c = torch.arange(D, device="cuda")[None]
    u = (c % 64) // 8
    off_main = (c // 64) * TR * 128 + (r // 8) * 1024 + (r % 8) * 128 + ((u ^ (r % 8)) * 16) + (c % 8) * 2
    ut = (c - main * 64) // 8
    off_tail = main * TR * 128 + (r // 8) * 256 + ut * 128 + (r % 8) * 16 + (c % 8) * 2
    off = torch.where(c < main * 64, off_main, off_tail) // 2
    buf = t.buf[kind * t.kind_stride:(kind + 1) * t.kind_stride].view(torch.bfloat16)
    tiles = buf.view(t.heads, t.tiles_per_head, -1)
    x = torch.zeros(t.heads, t.tiles_per_head, 128, D, device="cuda")
    x[:, :, :TR] = tiles[:, :, off.reshape(-1)].view(t.heads, t.tiles_per_head, TR, D).float()
    return x


def logical(t8):
    """The e4m3 tiles of a HeadTilesFp8 without the 128-byte swizzle, in the stand-in's layout."""
    r = torch.arange(128, device="cuda")[:, None]
    c = torch.arange(128, device="cuda")[None]
    idx = ((c // 16) ^ (r % 8)) * 16 + c % 16
    raw = t8.codes
    codes = raw.gather(-1, idx.expand(raw.shape)).view(E4M3)
    return types.SimpleNamespace(codes=codes, scales=t8.scales, map=t8.map, heads=t8.heads, head_dim=t8.head_dim,
                                 tiles_per_head=t8.tiles_per_head)


def _projected(osb, rows, tmap, kinds, H, D, seed, scale=1.0, rope=None):
    """Real bf16 head tiles from the projection GEMM (random activations and weights; RMSNorm on q / k)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    C = H * D
    K = 256
    a = (torch.randn(rows, K, device="cuda", generator=g) * scale).to(torch.bfloat16)
    w = (torch.randn(kinds * C, K, device="cuda", generator=g) / K ** 0.5).to(torch.bfloat16)
    bias = (torch.randn(kinds * C, device="cuda", generator=g) * 0.1).to(torch.bfloat16)
    t = osb.HeadTiles(rows, tmap, kinds, H, D, "cuda")
    osb.gemm_head_tiles(a, w, bias, t, nkinds=kinds)
    return t


@pytest.mark.parametrize("L,D,kinds,vp", [(3600, 72, 3, 3), (64, 72, 3, 3), (16, 64, 3, 3), (300, 72, 4, 2)])
def test_conversion_is_bit_equal_to_the_stand_in(L, D, kinds, vp):
    osb = _osb()
    tm = osb.tile_map(0, L, keys_only=(vp == 2))
    rows = (2 if L > 128 else 37) * L
    t = _projected(osb, rows, tm, kinds, 2, D, 0)
    t8 = osb.head_tiles_fp8(t, osb.HeadTilesFp8(t), v_period=vp, v_slot=vp - 1)
    lg = logical(t8)
    for k in range(kinds):
        x = bf16_tiles(t, k)
        codes, scales = F_.convert_v(x) if k % vp == vp - 1 else F_.convert_qk(x)
        assert torch.equal(lg.codes[k].view(torch.uint8), codes.view(torch.uint8)), k
        assert torch.equal(lg.scales[k], scales), k


CASES = {
    "spatial-S256": dict(L=256, nseq=4, D=72),
    "spatial-S3600": dict(L=3600, nseq=2, D=72),
    "temporal-T64-odd": dict(L=64, nseq=7, D=72),
    "temporal-T16-odd": dict(L=16, nseq=8 * 5 + 3, D=72),
    "temporal-T16-D64": dict(L=16, nseq=8 * 3 + 1, D=64),
    "cross-ragged-empty": dict(L=1024, nseq=3, D=72, Lk=300, kv_lens=[300, 77, 0]),
    "large-logits": dict(L=256, nseq=2, D=72, scale=30.0),
}


def _case(osb, c):
    L, nseq, D, H = c["L"], c["nseq"], c["D"], 4
    rows = L * nseq
    if "Lk" in c:
        qt = _projected(osb, rows, osb.tile_map(0, L, pack=False), 1, H, D, 1)
        kv = _projected(osb, c["Lk"] * nseq, osb.tile_map(0, c["Lk"], keys_only=True), 2, H, D, 2)
        q8 = osb.head_tiles_fp8(qt, osb.HeadTilesFp8(qt))
        kv8 = osb.head_tiles_fp8(kv, osb.HeadTilesFp8(kv), v_period=2, v_slot=1)
        kv_lens = torch.tensor(c["kv_lens"], dtype=torch.int32, device="cuda")
        kw = dict(q_kind=0, k_kind=0, v_kind=1, Lk=c["Lk"], num_seqs=nseq, kv_lens=kv_lens)
        return q8, kv8, kw, rows, c["Lk"] * nseq, c["Lk"], kv_lens
    t = _projected(osb, rows, osb.tile_map(0, L), 3, H, D, 3, scale=c.get("scale", 1.0))
    t8 = osb.head_tiles_fp8(t, osb.HeadTilesFp8(t), v_period=3, v_slot=2)
    return t8, t8, dict(Lk=L, num_seqs=nseq), rows, rows, L, None


@pytest.mark.parametrize("name", list(CASES))
def test_attention_against_dequantized_softmax(name):
    osb = _osb()
    c = CASES[name]
    q8, kv8, kw, rows, kv_rows, Lk, kv_lens = _case(osb, c)
    H, D = q8.heads, q8.head_dim
    out = torch.full((rows, H * D), float("nan"), dtype=torch.bfloat16, device="cuda")
    osb.attn_tiles_fp8(q8, kv8, out, **kw)
    again = torch.full_like(out, float("nan"))
    osb.attn_tiles_fp8(q8, kv8, again, **kw)
    torch.cuda.synchronize()
    assert torch.equal(out.view(torch.int16), again.view(torch.int16)), "a second call gives other bits"
    lq, lkv = logical(q8), logical(kv8)
    qseq, _ = F_._seq_pos(q8.map, rows, "cuda")
    kseq, kpos = F_._seq_pos(kv8.map, kv_rows, "cuda")
    exact, emu = A.tiles_reference(lq, lkv, rows, kv_rows, qseq, kseq, kpos, kw["num_seqs"], Lk,
                            None if kv_lens is None else kv_lens.cpu(), kw.get("q_kind", 0), kw.get("k_kind", 1),
                            kw.get("v_kind", 2))
    got = out.float().view(rows, H, D)
    assert torch.isfinite(got).all()
    r, r_emu = rel_l2(got, exact), rel_l2(emu, exact)
    print(f"[fp8 tiles gpu {name}] kernel {r:.3e}, P-emulation {r_emu:.3e}, ratio {r / r_emu:.3f}")
    if name == "large-logits":   # nearly one-hot rows: finite, and close to the emulation
        assert r < 3.0 * r_emu + 1e-2, (r, r_emu)
    else:
        assert r <= 1.1 * r_emu, (r, r_emu)
    if kv_lens is not None:
        assert not got[qseq == 2].any()


def test_output_scatter_is_the_unscattered_output():
    """Temporal attention with the frame-major output map, rows routed to two simulated ranks (mode 2: rank = frame //
    (T / 2)) held in local buffers: every row lands where the routing says, with the bits of the unscattered output."""
    osb = _osb()
    B, T, Sl, H, D = 1, 16, 40, 4, 72
    rows, C = B * T * Sl, H * D
    t = _projected(osb, rows, osb.tile_map(0, T), 3, H, D, 5)
    t8 = osb.head_tiles_fp8(t, osb.HeadTilesFp8(t), v_period=3, v_slot=2)
    om = osb.tile_map(1, T, Sl, T)
    plain = torch.zeros(rows, C, dtype=torch.bfloat16, device="cuda")
    osb.attn_tiles_fp8(t8, t8, plain, Lk=T, num_seqs=B * Sl, out_map=om)
    bufs = [torch.zeros(B * (T // 2) * 2 * Sl, C, dtype=torch.bfloat16, device="cuda") for _ in range(2)]
    sc = osb.make_scatter(2, 2, 0, T, Sl, [b.data_ptr() for b in bufs])
    osb.attn_tiles_fp8(t8, t8, None, Lk=T, num_seqs=B * Sl, out_map=om, out_scatter=sc, out_ld=C)
    torch.cuda.synchronize()
    tt = torch.arange(T, device="cuda")[:, None]
    ss = torch.arange(Sl, device="cuda")[None]
    src = (tt * Sl + ss).reshape(-1)
    peer = (tt // (T // 2)).expand(T, Sl).reshape(-1)
    dst = ((tt % (T // 2)) * (2 * Sl) + ss).reshape(-1)
    for p in range(2):
        sel = peer == p
        assert torch.equal(bufs[p][dst[sel]].view(torch.int16), plain[src[sel]].view(torch.int16))


@pytest.mark.parametrize("mlps", [False, True])
def test_xl_fp8_attention_at_the_benchmark_shape(mlps):
    """STDiT3-XL/2, full depth, 1x4x64x32x32, FP8 attention (and FP8 MLPs), against the fp32 oracle: at most 1.1x the
    error of the emulation reference, and the residual stream never jumps by more than 3x between consecutive blocks."""
    prod, oracle, cfg = stdit3_pair("xl")
    prod.enable_fp8_attention()
    if mlps:
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
        with A.fp8_attention(ob):
            if mlps:
                with R.fp8_mlps(ob):
                    emu = ob(**inp).float()
            else:
                emu = ob(**inp).float()
    r, _ = report(f"STDiT3-XL/2 64x32x32 FP8 attention{' + MLPs' if mlps else ''}", out, ref)
    r_emu, r_bf = rel_l2(emu, ref), rel_l2(floor, ref)
    print(f"[fp8 attn] emulation rel_l2={r_emu:.3e}, bf16 oracle rel_l2={r_bf:.3e}, ratio {r / r_emu:.3f}")
    print("[fp8 attn] residual stream rel_l2 after block k: " + " ".join(f"{k}:{e:.1e}" for k, e in enumerate(per_block)))
    assert torch.isfinite(out).all() and len(per_block) == 2 * cfg.depth
    for k in range(1, len(per_block)):
        assert per_block[k] < 3.0 * per_block[k - 1], (k, per_block[k - 1], per_block[k])
    assert r <= 1.1 * r_emu, (r, r_emu)


def test_graph_replay_and_disable():
    """STDiT3-XS/2 (4 heads of 72) with an x_mask and ragged text: the captured step replays to the eager bits, and
    disable_fp8_attention() gives the bits of a model that never enabled it."""
    prod, oracle, cfg = stdit3_pair("xs")
    plain = stdit3_pair("xs")[0]
    inp = stdit3_inputs(cfg, 2, 8, 16, 16, lens=[300, 21], device="cuda")
    xm = torch.ones(2, 8, dtype=torch.bool, device="cuda")
    xm[1, :3] = False
    with torch.no_grad():
        want_bf16 = plain(**inp, x_mask=xm)
        prod.enable_fp8_attention()
        eager = prod(**inp, x_mask=xm).clone()
        ref = oracle.cuda()(**inp, x_mask=xm)
    replay = prod.capture(**inp, x_mask=xm)
    got = replay(**inp, x_mask=xm).clone()
    torch.cuda.synchronize()
    assert torch.equal(got, eager)
    assert rel_l2(eager, ref) < 3e-2
    assert not torch.equal(eager, want_bf16)
    del replay
    prod.disable_fp8_attention()
    with torch.no_grad():
        back = prod(**inp, x_mask=xm)
    assert torch.equal(back, want_bf16)
