"""FP8 head-tile attention entries of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): a
torch restatement of `head_tiles_fp8` / `attn_tiles_fp8` (include/osb200.h, osb_head_tiles_fp8 / osb_attn_tiles_fp8)
with the kernels' refusals and the launch-count convention of tests/fake_osb200.py.

The e4m3 tiles are kept in their logical layout (the 128-byte swizzle of the real buffer is the kernels' business):
`codes` float8_e4m3fn [kinds, heads, tiles, 128, 128] (q / k: [tile row][channel]; v: [channel][position p], holding key
vt8_key(p) of the tile) and `scales` fp32 [kinds, heads, tiles, 128].  Tiles are filled from the dense rows of
tests/fake_osb200.HeadTiles through the binding's tile map, so rows no token maps to are zero, as in the real buffer.
Attention is computed from those operands as the kernel does: key tiles in order, scores in log2 units, online maximum,
P8 = e4m3(256 p), partial P8 V8 promoted as O = alpha O + s_v (.) partial, out = O / (256 l).

`install(monkeypatch)` adds these entries to tests/fake_osb200.py for one test."""
import torch

from tests import fake_osb200 as base
from tests.fake_osb200_fp8_attn import _e4m3, _scale, vt8_key

OsbError = base.OsbError
E4M3 = torch.float8_e4m3fn


def install(monkeypatch) -> None:
    for name in ("HeadTilesFp8", "head_tiles_fp8", "attn_tiles_fp8"):
        monkeypatch.setattr(base, name, globals()[name], raising=False)


def tile_index(m, rows: int, device):
    """(tile, row in tile) of every token row under tile map `m` (tiles.cuh tile_of_row)."""
    seq, pos = base._seq_pos(m, rows, device)
    if m.G > 1:
        return seq // m.G, (seq % m.G) * m.L + pos
    return seq * m.tps + pos // m.tile_rows, pos % m.tile_rows


def tiles_per_head(m, rows: int) -> int:
    seqs = rows // m.L
    return -(-seqs // m.G) if m.G > 1 else seqs * m.tps


class HeadTilesFp8:
    def __init__(self, tiles):
        if tiles.head_dim not in (64, 72):
            raise OsbError(f"FP8 head tiles are built for head_dim 64 and 72, not {tiles.head_dim}")
        self.src, self.map, self.kinds, self.heads, self.head_dim = tiles, tiles.map, tiles.kinds, tiles.heads, tiles.head_dim
        self.rows = tiles.rows
        self.tiles_per_head = tiles_per_head(tiles.map, tiles.rows)
        dev = tiles.dense.device
        self.codes = torch.zeros(self.kinds, self.heads, self.tiles_per_head, 128, 128, dtype=E4M3, device=dev)
        self.scales = torch.zeros(self.kinds, self.heads, self.tiles_per_head, 128, device=dev)


def bf16_tiles(tiles, kind: int) -> torch.Tensor:
    """fp32 [heads, tiles, 128, D]: the bf16 head tiles of one kind, rows past a tile's end zero."""
    H, D, dev = tiles.heads, tiles.head_dim, tiles.dense.device
    t, r = tile_index(tiles.map, tiles.rows, dev)
    x = torch.zeros(H, tiles_per_head(tiles.map, tiles.rows), 128, D, device=dev)
    x[:, t, r] = tiles.dense[kind].float().view(-1, H, D).transpose(0, 1)
    return x


def convert_qk(x: torch.Tensor):
    """[.., 128, D] fp32 -> (codes [.., 128, 128] e4m3, scales [.., 128]): per row."""
    s = _scale(x.abs().amax(-1))
    codes = torch.zeros(*x.shape[:-1], 128, dtype=E4M3, device=x.device)
    codes[..., : x.shape[-1]] = _e4m3(x / s[..., None])
    return codes, s


def convert_v(x: torch.Tensor):
    """[.., 128 keys, D] fp32 -> (codes [.., 128 channels, 128 positions] e4m3, scales [.., 128]): per channel over the
    tile, positions in the vt8 key order; channels past D zero with scale 1."""
    D = x.shape[-1]
    s = torch.ones(*x.shape[:-2], 128, device=x.device)
    s[..., :D] = _scale(x.abs().amax(-2))
    codes = torch.zeros(*x.shape[:-2], 128, 128, dtype=E4M3, device=x.device)
    keys = vt8_key(torch.arange(128, device=x.device))
    codes[..., :D, :] = _e4m3(x[..., keys, :] / s[..., None, :D]).transpose(-1, -2)
    return codes, s


def head_tiles_fp8(tiles, dst, *, kind0: int = 0, nkinds=None, v_period: int = 0, v_slot: int = 0):
    if dst.src is not tiles:
        raise OsbError("head_tiles_fp8: dst must be HeadTilesFp8(tiles) of the same bf16 tiles")
    nkinds = tiles.kinds - kind0 if nkinds is None else nkinds
    if not (0 <= kind0 and nkinds >= 1 and kind0 + nkinds <= tiles.kinds):
        raise OsbError(f"head_tiles_fp8: kinds [{kind0}, {kind0 + nkinds}) outside the {tiles.kinds} of the buffer")
    for k in range(nkinds):
        x = bf16_tiles(tiles, kind0 + k)
        is_v = v_period > 0 and k % v_period == v_slot
        dst.codes[kind0 + k], dst.scales[kind0 + k] = convert_v(x) if is_v else convert_qk(x)
    base._count("head_tiles_fp8", (nkinds, tiles.heads, dst.tiles_per_head))
    return dst


def v_in_key_order(codes: torch.Tensor) -> torch.Tensor:
    """[.., 128 channels, 128 positions] -> [.., 128 keys, 128 channels]."""
    out = torch.empty_like(codes.transpose(-1, -2))
    out[..., vt8_key(torch.arange(128, device=codes.device)), :] = codes.transpose(-1, -2)
    return out


def attn_tiles_fp8(q, kv, out, *, q_kind=0, k_kind=1, v_kind=2, Lk, num_seqs, kv_lens=None, softmax_scale=None,
                   out_scatter=None, out_ld=None, out_map=None):
    if not isinstance(q, HeadTilesFp8) or not isinstance(kv, HeadTilesFp8):
        raise OsbError("attn_tiles_fp8: q and kv must be HeadTilesFp8 buffers")
    base._need(out, torch.bfloat16, "out"); base._need(kv_lens, torch.int32, "kv_lens")
    assert out_scatter is None, "the CPU double writes local outputs only"
    m, km = q.map, kv.map
    if kv_lens is not None and m.G > 1:
        raise OsbError("attn_tiles_fp8: kv_lens applies to unpacked query maps only (G == 1); packed sequences see all Lk keys")
    if out_map is not None:
        assert out_map.key()[4:] == m.key()[4:] and out_map.L == m.L
    om = out_map if out_map is not None else m
    H, D, dev = q.heads, q.head_dim, out.device
    sc = (softmax_scale if softmax_scale is not None else D ** -0.5) * 1.4426950408889634
    nsets = -(-num_seqs // m.G) if m.G > 1 else num_seqs
    nq = nsets * m.tps
    BK, nkb = km.tile_rows, km.tps
    qt = torch.arange(nq, device=dev)
    sets, qpos = qt // m.tps, qt % m.tps
    keys = torch.full((nsets,), m.G * Lk if m.G > 1 else Lk, dtype=torch.long, device=dev)
    if kv_lens is not None:
        keys = torch.minimum(keys, kv_lens.to(dev).long().clamp(min=0))
    # query rows of every tile: sequence, position, validity, key range [lo, hi)
    r = torch.arange(128, device=dev)[None]
    if m.G > 1:
        g = r // m.L
        seq, pos = sets[:, None] * m.G + g, (r % m.L).expand(nq, 128)
        valid = (g < m.G) & (seq < num_seqs)
        lo, hi = g * Lk, g * Lk + Lk
    else:
        seq, pos = sets[:, None].expand(nq, 128), qpos[:, None] * m.tile_rows + r
        valid = (r < m.tile_rows) & (pos < m.L)
        lo, hi = torch.zeros_like(pos), keys[sets][:, None].expand(nq, 128)
    lo, hi = torch.where(valid, lo, 0), torch.where(valid, hi, 0)
    qd = q.codes[q_kind, :, :nq].float()                                  # [H, nq, 128, 128]
    sq = q.scales[q_kind, :, :nq] * sc                                    # [H, nq, 128]
    mrun = torch.full((H, nq, 128, 1), float("-inf"), device=dev)
    l = torch.zeros(H, nq, 128, 1, device=dev)
    o = torch.zeros(H, nq, 128, 128, device=dev)
    nkt = (keys + BK - 1) // BK
    for kb in range(nkb):
        ti = sets * nkb + kb
        kd = kv.codes[k_kind, :, ti].float()                              # [H, nq, 128, 128]
        vd = v_in_key_order(kv.codes[v_kind, :, ti]).float()
        s = (qd @ kd.transpose(-1, -2)) * sq[..., None] * kv.scales[k_kind, :, ti][:, :, None, :]
        slot = kb * BK + torch.arange(128, device=dev)
        ok = ((slot[None, None] < kb * BK + BK) & (slot[None, None] >= lo[..., None]) & (slot[None, None] < hi[..., None])
              & (kb < nkt[sets])[:, None, None])
        s = s.masked_fill(~ok[None], float("-inf"))
        mn = torch.maximum(mrun, s.amax(-1, keepdim=True))
        fin = mn != float("-inf")
        alpha = torch.where(fin, torch.exp2(mrun - torch.where(fin, mn, 0)), torch.ones_like(mn))
        p = torch.exp2(s - torch.where(fin, mn, 0))
        l = l * alpha + p.sum(-1, keepdim=True)
        part = _e4m3(256.0 * p).float() @ vd
        o = o * alpha + kv.scales[v_kind, :, ti][:, :, None, :] * part
        mrun = mn
    res = torch.where(l > 0, o / (256.0 * l), torch.zeros_like(o))[..., :D]   # [H, nq, 128, D]
    seq_v, pos_v = seq[valid], pos[valid]   # -> rows of `out`: tiles.cuh row_of_token under the output map
    orow = seq_v * om.L + pos_v if om.mode == 0 else ((seq_v // om.S) * om.T + pos_v) * om.S + seq_v % om.S
    out[orow] = res.permute(1, 2, 0, 3)[valid].reshape(-1, H * D).to(torch.bfloat16)
    base._count("attn_tiles_fp8", (num_seqs, m.L, Lk, H, D))
    return out
