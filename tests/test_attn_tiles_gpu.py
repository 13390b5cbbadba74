"""GPU parity of the head-tile path: projection GEMM with the head-tile epilogue (bias + per-head RMSNorm + RoPE fused,
osb_gemm_head_tiles) feeding the bulk-copy attention kernel (osb_attn_tiles), through the C ABI, against a plain fp32
torch restatement of Linear -> QK-RMSNorm -> RoPE -> softmax(QK^T)V on the same bf16 inputs.

Tolerances: the tile contents are ONE bf16 rounding of fp32 math (rel-L2 <= 2.5e-3, measured ~1.7e-3); attention adds
the bf16 rounding of P and of the output (<= 5e-3, measured ~2.5e-3), the same bars as tests/test_kernels_gpu.py."""
import math

import pytest
import torch

from tests.util import cross_case, rel_l2, self_case

pytestmark = pytest.mark.gpu


def _dev():
    if not torch.cuda.is_available():
        pytest.skip("needs a CUDA device")
    return torch.device("cuda:0")


@pytest.mark.parametrize("mode,B,T,S,H,D", [
    (0, 1, 3, 256, 4, 72),     # spatial, two q tiles sharing two resident key tiles (the STDiT3-XL shape)
    (1, 1, 64, 8, 4, 72),      # temporal T = 64: two sequences packed per tile, block-diagonal mask, RoPE
    (0, 2, 2, 128, 2, 72),     # one tile per sequence: the two slots work on different sets
    (0, 1, 2, 200, 2, 72),     # ragged last tile (72 of 128 rows), masked tail keys
    (0, 1, 1, 640, 2, 72),     # five key tiles > ring: streaming, online max
    (1, 2, 16, 12, 2, 72),     # eight sequences per tile: rows of one warp straddle sequences
    (1, 1, 17, 10, 2, 72),     # T = 17: 7 sequences per tile, 119 of 128 rows, odd tile count
    (1, 1, 100, 6, 2, 72),     # 64 < T <= 128: one 112-row tile per sequence
    (0, 1, 20, 256, 16, 72),   # 320 pairs over 148 CTAs: pair ranges straddle (sequence, head) groups
    (0, 1, 2, 256, 2, 64),     # head_dim 64 (no tail)
    (0, 1, 2, 256, 2, 128),    # head_dim 128 (two swizzled chunks)
])
def test_self_attention_tiles(mode, B, T, S, H, D):
    self_case(mode, B, T, S, H, D)


@pytest.mark.parametrize("mode,B,T,S,H,D", [
    (0, 1, 3, 256, 4, 72), (1, 1, 64, 8, 4, 72), (1, 2, 16, 16, 2, 72), (1, 1, 100, 6, 2, 72), (0, 1, 2, 256, 2, 128),
])
def test_general_epilogue_matches(mode, B, T, S, H, D):
    """Shapes the aligned fast path (staged tile image + bulk store, strided TMA view for the temporal case) takes by
    default, forced through the general per-row-store epilogue: both must produce the same tiles."""
    self_case(mode, B, T, S, H, D, general=True)


def test_temporal_odd_tile_count_and_batch():
    """Temporal fast path with an odd number of tiles per head (the pair's second CTA idles on the last tile) and B > 1
    (tile -> (batch, sequence group) decomposition of the strided TMA view)."""
    self_case(1, 3, 64, 6, 2, 72)      # 3 batches x 3 groups = 9 tiles
    self_case(1, 1, 32, 20, 2, 72)     # G = 4: 5 tiles


def test_softmax_large_logits_rescale():
    """Second key tile holds much larger logits than the first: the lazy-rescale branch (row max grows by > 2^8)."""
    import osb200 as osb

    dev = _dev()
    H, D, S = 2, 72, 256
    C = H * D
    g = torch.Generator().manual_seed(3)
    x = torch.randn(S, C, generator=g)
    x[128:] *= 6.0          # keys / queries of the second tile are larger -> logits jump
    x = x.to(torch.bfloat16).to(dev)
    w = (torch.randn(3 * C, C, generator=g) / math.sqrt(C) * 1.5).to(torch.bfloat16).to(dev)
    tm = osb.tile_map(0, S)
    tiles = osb.HeadTiles(S, tm, 3, H, D, dev)
    osb.gemm_head_tiles(x, w, None, tiles, nkinds=3)
    out = torch.empty(S, C, dtype=torch.bfloat16, device=dev)
    osb.attn_tiles(tiles, tiles, out, Lk=S, num_seqs=1)
    qkv = (x.float() @ w.float().t()).to(torch.bfloat16).float().view(S, 3, H, D)
    q, k, v = (qkv[:, i].permute(1, 0, 2) for i in range(3))
    logits = (q @ k.transpose(-1, -2)) * D ** -0.5 * 1.4426950408889634
    assert (logits[:, :, 128:].amax(-1) - logits[:, :, :128].amax(-1)).max() > 8.0, "case must exercise the rescale branch"
    ref = torch.nn.functional.scaled_dot_product_attention(q, k, v).permute(1, 0, 2).reshape(S, C)
    e = rel_l2(out.float(), ref)
    assert e < 5e-3, e


@pytest.mark.parametrize("B,N,Ly,lens,H", [
    (1, 512, 300, [260], 4),         # the STDiT3 cross-attention shape: 3 key tiles of 112
    (1, 10240, 300, [260], 4),       # 160 q pairs over 148 CTAs: key tiles stay resident across pairs of a head
    (2, 384, 300, [300, 7], 2),      # ragged text: 7 valid keys -> one key tile, 5 of 16 columns masked
    (2, 128, 120, [120, 33], 2),     # one q tile per sample: split mode with different key counts per slot
    (1, 256, 300, [0], 2),           # no valid key: zeros, not NaN
])
def test_cross_attention_tiles(B, N, Ly, lens, H):
    cross_case(B, N, Ly, lens, H)


def test_matches_register_path_kernel():
    """Same problem through the round-1 kernel (osb_attn_short on token-layout q/k/v) and through head tiles."""
    import osb200 as osb

    dev = _dev()
    B, T, S, H, D = 1, 4, 256, 4, 72
    C, R = H * D, B * T * S
    g = torch.Generator().manual_seed(5)
    x = torch.randn(R, C, generator=g).to(torch.bfloat16).to(dev)
    w = (torch.randn(3 * C, C, generator=g) / math.sqrt(C)).to(torch.bfloat16).to(dev)
    qn = (1.0 + 0.2 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    kn = (1.0 + 0.2 * torch.randn(D, generator=g)).to(torch.bfloat16).to(dev)
    qkv = osb.gemm(x, w)
    old = torch.empty(R, C, dtype=torch.bfloat16, device=dev)
    osb.attn_short(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], old, num_seqs=B * T, seqs_per_batch=T, q_strides=(T * S, S, 1),
                   k_strides=(T * S, S, 1), Lq=S, Lk=S, num_heads=H, head_dim=D, q_norm_w=qn, k_norm_w=kn)
    tiles = osb.HeadTiles(R, osb.tile_map(0, S), 3, H, D, dev)
    osb.gemm_head_tiles(x, w, None, tiles, nkinds=3, norm_w=(qn, kn, None))
    new = torch.empty_like(old)
    osb.attn_tiles(tiles, tiles, new, Lk=S, num_seqs=B * T)
    assert rel_l2(new.float(), old.float()) < 6e-3


@pytest.mark.parametrize("B,T,S,H", [(1, 64, 8, 4), (2, 64, 6, 2), (1, 32, 20, 2), (3, 16, 5, 2), (1, 17, 10, 2), (1, 100, 6, 2)])
def test_transposed_temporal_stream(B, T, S, H):
    """Temporal attention from a [B, S, T]-ordered token stream (what LN+modulate writes with osb_scatter mode 3): the QKV
    GEMM sees contiguous sequences (tile map mode 0, aligned epilogue when G*T == 128), the output rows are frame-major."""
    self_case(1, B, T, S, H, 72, transposed=True)


@pytest.mark.parametrize("mode", [1, 2, 3, 4])
def test_scatter_routing_on_one_gpu(mode):
    """osb_scatter row routing with the P 'ranks' simulated by P local buffers: every rank's LN+modulate call stores its
    rows into the buffer of the rank that consumes them; the buffers must equal the reference's all_to_all result
    (communications.py:8-18), or its transposed forms (modes 3, 4)."""
    import osb200 as osb

    dev = _dev()
    P = 1 if mode == 3 else 4
    B, T, S, C = 2, 8, 12, 64
    g = torch.Generator().manual_seed(9)
    full = torch.randn(B, T, S, C, generator=g).to(torch.bfloat16).to(dev)
    zeros = torch.zeros(1, C, dtype=torch.float32, device=dev)
    ref = torch.nn.functional.layer_norm(full.float(), (C,), eps=1e-6)
    Tl, Sl = T // P, S // P
    if mode in (1, 4):      # producers hold [B, Tl, S] (T-sharded), rank p ends up with every frame of its S/P columns
        bufs = [torch.full((B * T * Sl, C), float("nan"), dtype=torch.bfloat16, device=dev) for _ in range(P)]
        for r in range(P):
            x = full[:, r * Tl:(r + 1) * Tl].reshape(B * Tl * S, C).contiguous()
            osb.ln_modulate(x, zeros, zeros, group_rows=x.shape[0], scatter=osb.make_scatter(mode, P, r, Tl, S, bufs))
        for p in range(P):
            want = ref[:, :, p * Sl:(p + 1) * Sl]
            want = want if mode == 1 else want.transpose(1, 2)
            assert rel_l2(bufs[p].float().view(want.shape), want) < 3e-3
    elif mode == 2:         # producers hold [B, T, Sl] (S-sharded), rank p ends up with its T/P frames, all columns
        bufs = [torch.full((B * Tl * S, C), float("nan"), dtype=torch.bfloat16, device=dev) for _ in range(P)]
        for r in range(P):
            x = full[:, :, r * Sl:(r + 1) * Sl].reshape(B * T * Sl, C).contiguous()
            osb.ln_modulate(x, zeros, zeros, group_rows=x.shape[0], scatter=osb.make_scatter(2, P, r, T, Sl, bufs))
        for p in range(P):
            assert rel_l2(bufs[p].float().view(B, Tl, S, C), ref[:, p * Tl:(p + 1) * Tl]) < 3e-3
    else:                   # local transpose [B, T, S] -> [B, S, T]
        buf = torch.full((B * S * T, C), float("nan"), dtype=torch.bfloat16, device=dev)
        osb.ln_modulate(full.reshape(B * T * S, C), zeros, zeros, group_rows=B * T * S, scatter=osb.make_scatter(3, 1, 0, T, S, [buf]))
        assert rel_l2(buf.float().view(B, S, T, C), ref.transpose(1, 2)) < 3e-3


def test_attention_output_scatter_on_one_gpu():
    """The attention kernel's output rows routed by osb_scatter mode 2 (S-sharded temporal attention -> T-sharded token
    stream), 2 simulated ranks on one GPU: each 'rank' runs temporal attention on its S/P columns of the transposed stream
    and stores into the rank that owns the frame."""
    import osb200 as osb

    dev = _dev()
    P, B, T, S, H, D = 2, 1, 64, 8, 2, 72
    C, Sl, Tl = H * D, S // P, T // P
    g = torch.Generator().manual_seed(21)
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
    assert torch.equal(got, single), "sharded + routed output must be bit-identical to the single-GPU result"
