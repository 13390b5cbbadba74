"""GPU checks of the persistent schedule of osb_attn_tiles: every CTA walks a contiguous run of (head, set, query tile)
work items and keeps a set's key / value tiles resident while consecutive items share it.  The cases below make runs
start and end inside a set, cross head and sample boundaries, mix key counts per sample, overflow the stage ring
(head dim 128) and route the output rows to peer buffers; every result is checked against fp32 attention on the same
bf16 operands with the bars of tests/test_attn_tiles_gpu.py."""
import math

import pytest
import torch

from tests.util import rel_l2, self_case

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.parametrize("mode,B,T,S,H,D", [
    (0, 1, 41, 256, 16, 72),   # 1312 items: runs of ~9.9 items start on either query tile of a set and cross heads
    (1, 2, 64, 37, 8, 72),     # temporal, 37 packed tiles per head: runs cross head boundaries, no key reuse
    (0, 1, 20, 200, 8, 72),    # S = 200: ragged last query tile (72 rows), two key tiles in a four-stage ring
    (0, 1, 23, 300, 4, 64),    # head dim 64, three query and key tiles per set, 44-row last tiles
    (0, 1, 17, 256, 8, 128),   # head dim 128: two key tiles fill the two-stage ring and stay resident
])
def test_self_attention_runs(mode, B, T, S, H, D):
    _dev()
    nseq = B * T if mode == 0 else B * S
    L = S if mode == 0 else T
    items = H * (nseq * -(-L // 128) if mode == 0 else -(-nseq // (128 // L)))
    assert items > _sms(), "the case must give every CTA several items"
    self_case(mode, B, T, S, H, D, seed=7)


def _cross(B, N, Ly, lens, H, D, seed=13):
    import osb200 as osb

    dev = _dev()
    C = H * D
    g = torch.Generator().manual_seed(seed)
    xq = torch.randn(B * N, C, generator=g).to(torch.bfloat16).to(dev)
    y = torch.randn(B * Ly, C, generator=g).to(torch.bfloat16).to(dev)
    wq = (torch.randn(C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    wkv = (torch.randn(2 * C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    kv_lens = torch.tensor(lens, dtype=torch.int32, device=dev)
    qt = osb.HeadTiles(B * N, osb.tile_map(0, N), 1, H, D, dev)
    kt = osb.HeadTiles(B * Ly, osb.tile_map(0, Ly, keys_only=True), 2, H, D, dev)
    osb.gemm_head_tiles(xq, wq, None, qt, nkinds=1)
    osb.gemm_head_tiles(y, wkv, None, kt, nkinds=2)
    out = torch.full((B * N, C), float("nan"), dtype=torch.bfloat16, device=dev)
    osb.attn_tiles(qt, kt, out, q_kind=0, k_kind=0, v_kind=1, Lk=Ly, num_seqs=B, kv_lens=kv_lens)
    torch.cuda.synchronize()
    q = (xq.float() @ wq.float().t()).to(torch.bfloat16).float().view(B, N, H, D).permute(0, 2, 1, 3)
    kv = (y.float() @ wkv.float().t()).to(torch.bfloat16).float().view(B, Ly, 2, H, D)
    assert torch.isfinite(out.float()).all()
    for b in range(B):
        got = out[b * N:(b + 1) * N].float()
        n = min(lens[b], Ly)
        if n <= 0:
            assert (got == 0).all()
            continue
        k, v = kv[b, :n, 0].permute(1, 0, 2), kv[b, :n, 1].permute(1, 0, 2)
        ref = torch.nn.functional.scaled_dot_product_attention(q[b], k, v).permute(1, 0, 2).reshape(N, C)
        e = rel_l2(got, ref)
        assert e < 5e-3, (b, e)
    return out, (qt, kt, kv_lens)


@pytest.mark.parametrize("B,N,lens", [
    (3, 4096, [260, 7, 150]),         # 3, 1 and 2 key tiles: a run crossing samples must load the next sample's keys
    (4, 2000, [300, 0, 129, 260]),    # ragged last query tile per sample, an empty key set between two full ones
])
def test_cross_attention_runs_cross_samples(B, N, lens):
    H = 4
    items = H * B * -(-N // 128)
    assert items > _sms()
    _cross(B, N, 300, lens, H, 72)


def test_head_dim_128_reloads_keys():
    """Three text key tiles do not fit the two-stage ring of head dim 128: every item streams them again."""
    _cross(3, 3000, 300, [300, 200, 40], 4, 128)


def test_two_calls_identical_bits():
    import osb200 as osb

    out, (qt, kt, kv_lens) = _cross(3, 4096, 300, [260, 77, 300], 4, 72)
    again = torch.empty_like(out)
    osb.attn_tiles(qt, kt, again, q_kind=0, k_kind=0, v_kind=1, Lk=300, num_seqs=3, kv_lens=kv_lens)
    torch.cuda.synchronize()
    assert torch.equal(out, again)


def test_output_scatter_runs():
    """Temporal attention of 2 simulated ranks routed by osb_scatter mode 2, with more work items than CTAs per call:
    bit-identical to the single-GPU call."""
    import osb200 as osb

    dev = _dev()
    P, B, T, S, H, D = 2, 1, 64, 128, 8, 72
    C, Sl, Tl = H * D, S // P, T // P
    assert H * (B * Sl // 2) > _sms()
    g = torch.Generator().manual_seed(23)
    x = torch.randn(B, T, S, C, generator=g).to(torch.bfloat16).to(dev)
    w = (torch.randn(3 * C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    bufs = [torch.full((B * Tl * S, C), float("nan"), dtype=torch.bfloat16, device=dev) for _ in range(P)]
    single = torch.empty(B * T * S, C, dtype=torch.bfloat16, device=dev)
    tiles = osb.HeadTiles(B * S * T, osb.tile_map(0, T), 3, H, D, dev)
    osb.gemm_head_tiles(x.transpose(1, 2).reshape(B * S * T, C).contiguous(), w, None, tiles, nkinds=3)
    osb.attn_tiles(tiles, tiles, single, Lk=T, num_seqs=B * S, out_map=osb.tile_map(1, T, S, T))
    for r in range(P):
        xr = x[:, :, r * Sl:(r + 1) * Sl].transpose(1, 2).reshape(B * Sl * T, C).contiguous()
        tr = osb.HeadTiles(B * Sl * T, osb.tile_map(0, T), 3, H, D, dev)
        osb.gemm_head_tiles(xr, w, None, tr, nkinds=3)
        osb.attn_tiles(tr, tr, None, Lk=T, num_seqs=B * Sl, out_map=osb.tile_map(1, T, Sl, T),
                       out_scatter=osb.make_scatter(2, P, r, T, Sl, bufs), out_ld=C)
    got = torch.cat([b.view(B, Tl, S, C) for b in bufs], 1).reshape(B * T * S, C)
    assert torch.equal(got, single)
    # and the single call itself against fp32 attention
    qkv = (x.float().view(B * T * S, C) @ w.float().t()).to(torch.bfloat16).float().view(B, T, S, 3, H, D)
    q, k, v = (qkv[..., i, :, :].permute(0, 2, 3, 1, 4) for i in range(3))   # [B, S, H, T, D]
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).permute(0, 3, 1, 2, 4).reshape(B * T * S, C)
    assert rel_l2(single.float(), ref) < 5e-3
