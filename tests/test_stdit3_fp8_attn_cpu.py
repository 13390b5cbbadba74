"""The FP8 (e4m3) head-tile attention of STDiT3 on the CPU: the stand-in entries of tests/fake_osb200.py against
the written contract (conversion codes and scales, attention against fp32 softmax on the dequantized tiles) on every set
shape the model uses, the host-side STDiT3 with `enable_fp8_attention()` against the FP8-emulation reference
(tests/stdit3_fp8_attn_ref.py), `disable_fp8_attention()`, the refusals, sequence parallelism on two gloo ranks and the
ctypes mirrors of the new structs."""
import ctypes
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests import stdit3_fp8_attn_ref as A
from tests.models import stdit3_inputs, stdit3_pair
from tests.util import rel_l2

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _tiles(osb, rows, tmap, kinds, H, D, seed, spread=True):
    g = torch.Generator().manual_seed(seed)
    t = osb.HeadTiles(rows, tmap, kinds, H, D, "cpu")
    x = torch.randn(kinds, rows, H * D, generator=g)
    if spread:   # rows and channels over several decades, one all-zero row
        x = x * torch.logspace(-2, 1, rows)[torch.randperm(rows, generator=g)][None, :, None]
        x[:, 3] = 0.0
    t.dense.copy_(x.to(torch.bfloat16))
    return t


@pytest.mark.parametrize("L,D", [(300, 72), (16, 64)])
def test_conversion_follows_the_contract(fake_osb, L, D):
    """q / k per row, v per (tile, channel) over the tile's rows, transposed in the vt8 key order; zero rows give scale 1."""
    tm = fake_osb.tile_map(0, L)
    rows, H = 4 * L, 2
    t = _tiles(fake_osb, rows, tm, 3, H, D, 0)
    t8 = fake_osb.head_tiles_fp8(t, fake_osb.HeadTilesFp8(t), v_period=3, v_slot=2)
    ti, r = F_.tile_index(tm, rows, "cpu")
    for kind in (0, 1):
        x = t.dense[kind].float().view(rows, H, D)
        q, s = R.quantize(x)
        got = t8.codes[kind][:, ti, r].transpose(0, 1)                     # [rows, H, 128]
        assert torch.equal(got[..., :D].double(), q) and not got[..., D:].float().any()
        assert torch.equal(t8.scales[kind][:, ti, r].t(), s)
        assert torch.all(s[3] == 1.0)
    x = t.dense[2].float().view(rows, H, D)
    ntiles = t8.tiles_per_head
    amax = torch.zeros(ntiles, H, D).scatter_reduce(0, ti[:, None, None].expand_as(x), x.abs(), "amax")
    sv = torch.where(amax > 0, amax / 448.0, torch.ones_like(amax))
    assert torch.equal(t8.scales[2][..., :D].permute(1, 0, 2), sv) and torch.all(t8.scales[2][..., D:] == 1.0)
    assert torch.equal(A.dequantized(t8, 2, rows, True), (R.e4m3_round(x / sv[ti]) * sv[ti].double()))


CASES = {
    "spatial-3-tiles": dict(L=300, nseq=2, D=72),
    "temporal-T64": dict(L=64, nseq=5, D=72),
    "temporal-T16": dict(L=16, nseq=19, D=64),
    "temporal-transposed": dict(L=16, nseq=12, D=72, transposed=True),
    "cross-ragged": dict(L=200, nseq=3, D=72, Lk=300, kv_lens=[300, 77, 0]),
}


@pytest.mark.parametrize("name", list(CASES))
def test_attention_follows_dequantized_softmax(fake_osb, name):
    c = CASES[name]
    L, nseq, D, H = c["L"], c["nseq"], c["D"], 2
    rows = L * nseq
    out_map = None
    if "Lk" in c:   # cross: queries unpacked, keys of the text tiles
        qt = _tiles(fake_osb, rows, fake_osb.tile_map(0, L, pack=False), 1, H, D, 1)
        kv = _tiles(fake_osb, c["Lk"] * nseq, fake_osb.tile_map(0, c["Lk"], keys_only=True), 2, H, D, 2)
        q8 = fake_osb.head_tiles_fp8(qt, fake_osb.HeadTilesFp8(qt))
        kv8 = fake_osb.head_tiles_fp8(kv, fake_osb.HeadTilesFp8(kv), v_period=2, v_slot=1)
        kv_lens = torch.tensor(c["kv_lens"], dtype=torch.int32)
        kw = dict(q_kind=0, k_kind=0, v_kind=1, Lk=c["Lk"], num_seqs=nseq, kv_lens=kv_lens)
        kv_rows, Lk = c["Lk"] * nseq, c["Lk"]
    else:
        qt = _tiles(fake_osb, rows, fake_osb.tile_map(0, L), 3, H, D, 3)
        q8 = kv8 = fake_osb.head_tiles_fp8(qt, fake_osb.HeadTilesFp8(qt), v_period=3, v_slot=2)
        kw = dict(Lk=L, num_seqs=nseq)
        kv_rows, Lk, kv_lens = rows, L, None
        if c.get("transposed"):   # tiles from the [B, S, T] stream, output rows frame-major [B, T, S]
            S = nseq // 2
            out_map = fake_osb.tile_map(1, L, S, L)
            kw["out_map"] = out_map
    out = torch.full((rows, H * D), float("nan"), dtype=torch.bfloat16)
    fake_osb.attn_tiles_fp8(q8, kv8, out, **kw)
    qseq, _ = fake_osb._seq_pos(q8.map, rows, "cpu")
    kseq, kpos = fake_osb._seq_pos(kv8.map, kv_rows, "cpu")
    exact, emu = A.tiles_reference(q8, kv8, rows, kv_rows, qseq, kseq, kpos, nseq, Lk, kv_lens, kw.get("q_kind", 0),
                            kw.get("k_kind", 1), kw.get("v_kind", 2))
    if out_map is not None:   # row (seq, pos) of the tiles' stream lives at the frame-major row of `out`
        so, po = fake_osb._seq_pos(out_map, rows, "cpu")
        inv = torch.empty(rows, dtype=torch.long)
        inv[so * L + po] = torch.arange(rows)
        got = out[inv[qseq * L + torch.arange(rows) % L]].float().view(rows, H, D)
    else:
        got = out.float().view(rows, H, D)
    assert not got.isnan().any()
    r, r_emu = rel_l2(got, exact), rel_l2(emu, exact)
    print(f"[fp8 tiles {name}] stand-in {r:.3e}, P-emulation {r_emu:.3e}")
    assert r < 1.25 * r_emu + 1e-3, (r, r_emu)
    if kv_lens is not None:   # an empty key set writes zeros, as osb_attn_tiles does
        assert not got[qseq == 2].any()


@pytest.mark.parametrize("which,mlps", [("xs72", False), ("xs64", False), ("xs64", True)])
def test_host_stdit3_fp8_attention_follows_the_emulation(fake_osb, which, mlps):
    """The product with FP8 attention (and FP8 MLPs) on the stand-in, against the fp32 oracle: at most 1.1x further away
    than the emulation reference (the bf16 oracle with its attentions, and MLPs, at the FP8 rounding points), plain and
    with an x_mask and ragged text."""
    prod, oracle, cfg = stdit3_pair("xs" if which == "xs72" else which, device="cpu")
    prod.enable_fp8_attention()
    if mlps:
        prod.enable_fp8()
    inp = stdit3_inputs(cfg, 2, 4, 8, 8, lens=[cfg.model_max_length, 9])
    xm = torch.ones(2, 4, dtype=torch.bool)
    xm[1, 1:3] = False
    ob = stdit3_pair("xs" if which == "xs72" else which, device="cpu")[1].to(torch.bfloat16)
    for kw in ({}, {"x_mask": xm}):
        fake_osb.reset()
        with torch.no_grad():
            ref = oracle(**inp, **kw)
            out = prod(**inp, **kw)
            with A.fp8_attention(ob):
                if mlps:
                    with R.fp8_mlps(ob):
                        emu = ob(**inp, **kw).float()
                else:
                    emu = ob(**inp, **kw).float()
            floor = ob(**inp, **kw).float()
        r_emu, r_out, r_bf = rel_l2(emu, ref), rel_l2(out, ref), rel_l2(floor, ref)
        print(f"[fp8 attn host {which} mlps={mlps}] {'x_mask' if kw else 'plain'}: product {r_out:.3e}, "
              f"emulation {r_emu:.3e}, bf16 oracle {r_bf:.3e}")
        assert r_out < 1.1 * r_emu and r_emu > r_bf, (r_out, r_emu, r_bf)
        names = [c[0] for c in fake_osb.calls]
        nb = 2 * cfg.depth
        assert names.count("attn_tiles_fp8") == 2 * nb and names.count("attn_tiles") == 0
        # per block: the q | k | v conversion and the cross-attention q; once per forward: all blocks' text k | v
        assert names.count("head_tiles_fp8") == 2 * nb + 1


def test_disable_fp8_attention_restores_the_bf16_path(fake_osb):
    prod, _, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, 1, 4, 8, 8)
    with torch.no_grad():
        fake_osb.reset()
        before = prod(**inp)
        calls_before = list(fake_osb.calls)
        prod.enable_fp8_attention()
        fp8 = prod(**inp)
        assert any(k[0] == "fp8attn" for k in prod._cache)
        prod.disable_fp8_attention()
        fake_osb.reset()
        after = prod(**inp)
    assert not torch.equal(before, fp8)
    assert torch.equal(before, after)
    assert fake_osb.calls == calls_before
    assert not any(k[0] == "fp8attn" for k in prod._cache)


def test_head_layout_refusals(fake_osb):
    """FP8 attention refuses head sizes it is not built for; the forward refuses, with or without FP8 attention, any
    head layout the head tiles are not built for, before its first launch."""
    from opensora.models.stdit.stdit3 import STDiT3, STDiT3Config

    with torch.device("meta"):
        m = STDiT3(STDiT3Config(depth=1, hidden_size=256, num_heads=2, caption_channels=128, model_max_length=8))
    with pytest.raises(ValueError, match="head sizes 72 and 64"):
        m.enable_fp8_attention()                    # 2 heads of 128
    assert m._fp8_attn is False
    _, _, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, 1, 2, 4, 4)
    # head tiles need an even head count (3 heads of 72, with and without FP8 attention) and a head size they are built
    # for (4 heads of 96): the forward refuses both before its first launch
    for heads, hidden, fp8 in ((3, 216, False), (3, 216, True), (4, 384, False)):
        bad = STDiT3(STDiT3Config(depth=1, hidden_size=hidden, num_heads=heads, caption_channels=cfg.caption_channels,
                                  model_max_length=cfg.model_max_length)).to(torch.bfloat16)
        if fp8:
            bad.enable_fp8_attention()
        fake_osb.reset()
        with pytest.raises(ValueError, match=f"{heads} heads of {hidden // heads}"), torch.no_grad():
            bad(**inp)
        assert fake_osb.launch_count() == 0


def _sp_worker(rank, world, port, ret):
    import sys

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        torch.manual_seed(0)
        prod, _, cfg = stdit3_pair("xs", device="cpu")
        prod.enable_fp8_attention()
        # 16 x 16 latent: S = 64 (spatial sequences packed in pairs), T = 4 (temporal sequences packed 32 per tile): each
        # rank's S / 2 = 32 columns fill whole temporal tiles, so both runs group the same sequences into one v scale
        inp = stdit3_inputs(cfg, 2, 4, 16, 16, lens=[cfg.model_max_length, 9])
        xm = torch.ones(2, 4, dtype=torch.bool)
        xm[1, 2:] = False
        with torch.no_grad():
            single = prod(**inp, x_mask=xm)
            prod.enable_sequence_parallel(dist.group.WORLD)
            sharded = prod(**inp, x_mask=xm)
            prod.enable_sequence_parallel(None)
        ret[rank] = bool(torch.equal(single, sharded))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sequence_parallel_fp8_attention_world2_is_bit_identical():
    """With FP8 attention, the T-sharded model on two gloo ranks (all-to-all around every temporal attention, the mode-1
    output map) reproduces the single-rank output bit for bit."""
    port = 29500 + (os.getpid() + 11) % 2000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_sp_worker, args=(2, port, ret), nprocs=2, join=True)
    assert ret.get(0) is True and ret.get(1) is True


def test_fp8_tile_structs_match_header():
    import subprocess
    import tempfile

    import osb200

    fields = [
        ("sizeof(osb_tiles_fp8)", ctypes.sizeof(osb200.TilesFp8)),
        ("sizeof(osb_head_tiles_fp8_args)", ctypes.sizeof(osb200.HeadTilesFp8Args)),
        ("offsetof(osb_head_tiles_fp8_args, dst)", osb200.HeadTilesFp8Args.dst.offset),
        ("offsetof(osb_head_tiles_fp8_args, v_slot)", osb200.HeadTilesFp8Args.v_slot.offset),
        ("sizeof(osb_attn_tiles_fp8_operands)", ctypes.sizeof(osb200.AttnTilesFp8Operands)),
        ("offsetof(osb_attn_tiles_fp8_operands, kv_head_tiles)", osb200.AttnTilesFp8Operands.kv_head_tiles.offset),
    ]
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){\n')
            for expr, _ in fields:
                f.write(f'printf("%zu\\n", (size_t)({expr}));\n')
            f.write("return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(ROOT, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_new_entry_points_refuse_before_init():
    import osb200

    rc = osb200._lib.osb_head_tiles_fp8(ctypes.byref(osb200.HeadTilesFp8Args()), None)
    assert rc != 0 and "osb_init" in osb200.last_error()
    rc = osb200._lib.osb_attn_tiles_fp8(ctypes.byref(osb200.AttnTilesArgs()), ctypes.byref(osb200.AttnTilesFp8Operands()),
                                        None)
    assert rc != 0 and "osb_init" in osb200.last_error()
