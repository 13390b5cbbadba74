"""FP8-emulation reference of the STDiT3 FP8 attention path (include/osb200.h, osb_head_tiles_fp8 / osb_attn_tiles_fp8),
for the tests.

The oracle STDiT3 (`oracle/stdit3_oracle.py`), typically run in bf16, with every self-attention (spatial and temporal)
and every cross-attention computed in fp32 on dequantized operands, rounded where the product rounds:
- q and k after RMSNorm and RoPE (in the oracle's dtype), per (token, head);
- v per (key tile, head, channel): key tiles of 128 consecutive keys of a sequence, or the G = 128 // L short sequences
  packed into one tile when L <= 64 (temporal attention at T <= 64, spatial attention at S <= 64);
- P as e4m3(256 p) / 256 with p relative to the final row maximum, normalised by the fp32 sum of the unquantized p.
The kernel quantizes P against the running maximum of its key tiles, and its text-key tiles also hold the padding tokens
past a sample's text length (their v rows count in the tile's scale, the oracle never sees them), so this is not the
kernel's arithmetic bit for bit; it is the same kind of yardstick the other FP8 references are.
`fp8_attention(oracle)` patches one oracle for the duration of a `with` and composes with fp8_ref.fp8_mlps."""
import contextlib

import torch

from tests import fake_osb200 as F_
from tests import fp8_ref as R
from tests.mmdit_fp8_attn_ref import attention_from_operands


def key_tiles(n_seq: int, L: int, device) -> torch.Tensor:
    """[n_seq, L] key tile of every (sequence, position) under the head-tile map of self-attention over L tokens."""
    seq = torch.arange(n_seq, device=device)[:, None]
    pos = torch.arange(L, device=device)[None]
    if L <= 64:
        return (seq // (128 // L)).expand(n_seq, L)
    return seq * (-(-L // 128)) + pos // 128


def qdq_v(v: torch.Tensor, tiles: torch.Tensor) -> torch.Tensor:
    """v [n, H, L, D] -> dequantized e4m3 with one scale per (key tile, head, channel); tiles [n, L]."""
    n, H, L, D = v.shape
    vt = v.float().permute(0, 2, 1, 3).reshape(n * L, H, D)
    idx = tiles.reshape(-1)
    amax = torch.zeros(int(idx.max()) + 1, H, D, device=v.device).scatter_reduce(
        0, idx[:, None, None].expand_as(vt), vt.abs(), "amax")
    s = torch.where(amax > 0, amax / R.E4M3_MAX, torch.ones_like(amax))[idx]
    return (R.e4m3_round(vt / s).float() * s).view(n, L, H, D).permute(0, 2, 1, 3)


def _self_attention(attn):
    def forward(x):
        B, N, C = x.shape
        qkv = attn.qkv(x).view(B, N, 3, attn.num_heads, attn.head_dim).permute(2, 0, 3, 1, 4)
        q, k, v = qkv.unbind(0)
        q, k = attn.q_norm(q), attn.k_norm(k)
        if attn.rotary_emb is not None:
            q, k = attn.rotary_emb(q), attn.rotary_emb(k)
        o = attention_from_operands(R.qdq(q.float()), R.qdq(k.float()), qdq_v(v, key_tiles(B, N, x.device)), attn.scale)
        return attn.proj(o.to(x.dtype).transpose(1, 2).reshape(B, N, C))
    return forward


def _cross_attention(ca):
    def forward(x, cond, y_lens):
        B, N, C = x.shape
        q = ca.q_linear(x).view(B, N, ca.num_heads, ca.head_dim)
        kv = ca.kv_linear(cond).view(-1, 2, ca.num_heads, ca.head_dim)
        outs, off = [], 0
        for b in range(B):
            n = int(y_lens[b])
            k, v = kv[off:off + n, 0].transpose(0, 1), kv[off:off + n, 1].transpose(0, 1)   # [H, n, D]
            off += n
            qb = q[b].transpose(0, 1)
            if n == 0:
                outs.append(torch.zeros(N, C, dtype=x.dtype, device=x.device))
                continue
            vd = qdq_v(v[None], (torch.arange(n, device=x.device) // 128)[None])[0]
            o = attention_from_operands(R.qdq(qb.float()), R.qdq(k.float()), vd, ca.head_dim ** -0.5)
            outs.append(o.to(x.dtype).transpose(0, 1).reshape(N, C))
        return ca.proj(torch.stack(outs, 0))
    return forward


@contextlib.contextmanager
def fp8_attention(oracle):
    """Run every attention of the oracle STDiT3's blocks at the FP8 rounding points."""
    blocks = [b for pair in zip(oracle.spatial_blocks, oracle.temporal_blocks) for b in pair]
    for b in blocks:
        b.attn.forward = _self_attention(b.attn)
        b.cross_attn.forward = _cross_attention(b.cross_attn)
    try:
        yield oracle
    finally:
        for b in blocks:
            del b.attn.forward
            del b.cross_attn.forward


def dequantized(t8, kind, rows, is_v):
    """fp64 [rows, H, D] values of one kind read back from the e4m3 tiles through the tile map."""
    ti, r = F_.tile_index(t8.map, rows, t8.codes.device)
    codes = t8.codes[kind].double()
    if is_v:
        codes = F_.v_in_key_order(t8.codes[kind]).double()
        x = codes[:, ti, r, : t8.head_dim] * t8.scales[kind][:, ti, : t8.head_dim].double()
    else:
        x = codes[:, ti, r, : t8.head_dim] * t8.scales[kind][:, ti, r, None].double()
    return x.transpose(0, 1)


def tiles_reference(t8, kv8, q_rows, kv_rows, qseq, kseq, kpos, num_seqs, Lk, kv_lens, q_kind, k_kind, v_kind):
    """(exact fp32 softmax, the P-emulation) on the dequantized e4m3 operands, per output token row [rows, H, D]."""
    q = dequantized(t8, q_kind, q_rows, False).float()
    k = dequantized(kv8, k_kind, kv_rows, False).float()
    v = dequantized(kv8, v_kind, kv_rows, True).float()
    H, D = t8.heads, t8.head_dim
    exact = torch.zeros(q_rows, H, D, device=q.device)
    emu = torch.zeros(q_rows, H, D, device=q.device)
    for s_ in range(num_seqs):
        rq = (qseq == s_).nonzero().flatten()
        rk = (kseq == s_).nonzero().flatten()
        rk = rk[kpos[rk].argsort()]
        n = Lk if kv_lens is None else min(int(kv_lens[s_]), Lk)
        if n <= 0:
            continue
        rk = rk[:n]
        qq, kk, vv = q[rq].transpose(0, 1), k[rk].transpose(0, 1), v[rk].transpose(0, 1)
        sc = qq @ kk.transpose(-1, -2) * D ** -0.5
        exact[rq] = (torch.softmax(sc.double(), -1).float() @ vv).transpose(0, 1)
        emu[rq] = attention_from_operands(qq, kk, vv, D ** -0.5).transpose(0, 1)
    return exact, emu
