"""CPU stand-in for the `osb200` binding, used ONLY by the host-logic tests (`-m "not gpu"`).

TEST INFRASTRUCTURE, not a fallback: the product never imports this module, and `osb200` itself still refuses to run
without CUDA.  The host side of the drop-in (opensora/models/*, utils/sampling.py) is a few thousand lines of shape /
stride / caching logic around the C ABI calls; this double implements the *documented contract* of every binding
function (include/osb200.h, open-sora_b200/osb200/__init__.py docstrings) with plain torch ops so that this logic can
be executed on the CPU box and compared with the oracle: patch embedding, modulation tables and `x_mask` indexing,
the packed kv projection, the row-stride conventions of spatial / temporal / cross attention, sequence-parallel
transpositions (gloo, world size 2), VAE padding / up-sampling / tiling arithmetic.

Rounding points mirror the kernels (fp32 math, one rounding to bf16 per op; attention rounds q-hat, k-hat and P to
bf16) so tolerances in the host tests are the same bf16 noise floors as on the GPU.  Tests install it with the
`fake_osb` fixture of tests/conftest.py (`sys.modules["osb200"]` for the duration of one test)."""
import math

import torch
import torch.nn.functional as F

EPI_BIAS, EPI_BIAS_GELU_TANH, EPI_BIAS_GATE_RES = 0, 1, 2
ATTN_IMPL = 0
_launches = 0
calls = []   # (name, detail) log, so tests can assert how the host code drives the boundary


class OsbError(RuntimeError):
    pass


def _count(name, detail=None, launches=1):
    global _launches
    _launches += launches
    calls.append((name, detail))


def reset():
    global _launches
    _launches = 0
    calls.clear()


def launch_count() -> int:
    return _launches


def init(device=None) -> None:
    pass


def start_profile():
    pass


def stop_profile():
    return []


def require_cuda_bf16(t, what: str) -> None:
    if t.dtype != torch.bfloat16:   # the dtype half of the contract still holds on the CPU double
        raise OsbError(f"{what} (osb200) runs in bfloat16 only")


def _need(t, dtype, name):
    if t is None:
        return
    if t.dtype != dtype:
        raise OsbError(f"{name} must be {dtype}, got {t.dtype}")
    if t.dim() >= 1 and t.stride(-1) != 1 and t.shape[-1] != 1:
        raise OsbError(f"{name} must have unit stride in the last dimension")


def _epilogue_shapes(fn, M, N, out_cols, out, bias, residual, gate, group_rows, mod_index):
    """The binding's extent checks of the optional GEMM operands (osb200._epilogue_shapes), raised before any math."""
    if out is not None and tuple(out.shape) != (M, out_cols):
        raise OsbError(f"{fn}: out must be [{M}, {out_cols}], got {tuple(out.shape)}")
    if bias is not None and tuple(bias.shape) != (N,):
        raise OsbError(f"{fn}: bias must be [{N}], got {tuple(bias.shape)}")
    if residual is not None and tuple(residual.shape) != (M, N):
        raise OsbError(f"{fn}: residual must be [{M}, {N}], got {tuple(residual.shape)}")
    groups = -(-M // (group_rows if group_rows > 0 else M))
    if gate is not None and (gate.dim() != 2 or gate.shape[1] != N or (mod_index is None and gate.shape[0] < groups)):
        raise OsbError(f"{fn}: gate must be [G, {N}] with G >= {groups} row groups, got {tuple(gate.shape)}")
    if mod_index is not None and (mod_index.dim() != 1 or mod_index.shape[0] < groups):
        raise OsbError(f"{fn}: mod_index must be 1-D with at least {groups} entries, got {tuple(mod_index.shape)}")


def _groups(rows, group_rows, mod_index, device):
    g = torch.arange(rows, device=device) // max(int(group_rows), 1)
    if mod_index is not None:
        g = mod_index.long()[g]
    return g


class Scatter:
    def __init__(self, mode, P, rank, I, J, peers):
        self.mode, self.P, self.rank, self.I, self.J, self.peers = mode, P, rank, I, J, peers


def make_scatter(mode, P, rank, I, J, peer_bufs):
    """The double routes rows into torch tensors (`peer_bufs`) instead of raw pointers; only what one process can do on its
    own is supported: P == 1 (mode 3, the local transpose)."""
    return Scatter(mode, P, rank, I, J, peer_bufs)


def ln_modulate(x, shift, scale, *, group_rows: int, mod_index=None, eps: float = 1e-6, out=None, scatter=None):
    if scatter is not None:
        assert scatter.mode == 3 and scatter.P == 1, "the CPU double only routes the local transpose"
        y = ln_modulate(x, shift, scale, group_rows=group_rows, mod_index=mod_index, eps=eps)
        I, J = scatter.I, scatter.J
        B = x.shape[0] // (I * J)
        scatter.peers[0].copy_(y.view(B, I, J, -1).transpose(1, 2).reshape(x.shape[0], -1))
        return None
    _need(x, torch.bfloat16, "x"); _need(shift, torch.float32, "shift"); _need(scale, torch.float32, "scale")
    _need(mod_index, torch.int32, "mod_index")
    assert x.dim() == 2 and x.is_contiguous()
    assert shift.dim() == 2 and scale.dim() == 2 and shift.stride(0) == scale.stride(0)
    rows, C = x.shape
    if C % 8 or C > 8192:
        raise OsbError(f"osb_ln_modulate failed (-1): C must be a multiple of 8 and <= 8192 (got {C})")
    xf = x.float()
    mu = xf.mean(-1, keepdim=True)
    var = (xf - mu).pow(2).mean(-1, keepdim=True)
    g = _groups(rows, group_rows, mod_index, x.device)
    y = ((xf - mu) * torch.rsqrt(var + eps) * (1.0 + scale[g]) + shift[g]).to(torch.bfloat16)
    _count("ln_modulate", (rows, x.shape[1]))
    if out is None:
        return y
    out.copy_(y)
    return out


# Accumulation dtype of the GEMM / convolution stand-ins.  fp32 by default; a test that compares two decompositions of the
# SAME computation (e.g. a frame-sharded convolution against the whole one) switches to fp64, where the summation order of
# the CPU kernels can no longer flip a bf16 rounding, so the comparison can be bit-exact.
ACC_DTYPE = torch.float32


def gemm(a, w, bias=None, *, epilogue: int = EPI_BIAS, residual=None, gate=None, group_rows: int = 0, mod_index=None,
         out=None, cta_group: int = 0, block_n: int = 0):
    for t, n in ((a, "a"), (w, "w"), (bias, "bias"), (residual, "residual"), (out, "out")):
        _need(t, torch.bfloat16, n)
    _need(gate, torch.float32, "gate"); _need(mod_index, torch.int32, "mod_index")
    if a.dim() != 2 or w.dim() != 2 or a.shape[1] != w.shape[1]:
        raise OsbError(f"gemm: a [M, K] and w [N, K] expected, got {tuple(a.shape)} and {tuple(w.shape)}")
    M, K = a.shape
    N = w.shape[0]
    _epilogue_shapes("gemm", M, N, N, out, bias, residual, gate, group_rows, mod_index)
    if K % 8 or N % 8:
        raise OsbError(f"osb_gemm_bf16 failed (-1): osb_gemm_bf16: K and N must be multiples of 8 (K {K} N {N})")
    acc = a.to(ACC_DTYPE) @ w.to(ACC_DTYPE).t()
    if bias is not None:
        acc = acc + bias.to(ACC_DTYPE)
    if epilogue == EPI_BIAS_GELU_TANH:
        acc = F.gelu(acc, approximate="tanh")
    elif epilogue == EPI_BIAS_GATE_RES:
        if gate is not None:
            g = _groups(M, group_rows if group_rows > 0 else M, mod_index, a.device)
            acc = acc * gate[g]
        if residual is not None:
            acc = acc + residual.to(ACC_DTYPE)
    y = acc.to(torch.bfloat16)
    _count("gemm", (M, N, K, epilogue))
    if out is None:
        return y
    out.copy_(y)   # `out` may alias `residual` (in-place residual stream): y is already materialised
    return out


def _rms(x, w, eps):
    return x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * w


def _rope_interleaved(x, cos, sin):   # x [..., L, D], tables [L, D/2]: pairs (2i, 2i+1)
    x1, x2 = x[..., 0::2], x[..., 1::2]
    return torch.stack((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1).flatten(-2)


def _rope_half(x, cos, sin):          # pairs (i, i + D/2)
    h = x.shape[-1] // 2
    x1, x2 = x[..., :h], x[..., h:]
    return torch.cat((x1 * cos - x2 * sin, x2 * cos + x1 * sin), dim=-1)


def attn_short(q, k, v, out, *, num_seqs: int, seqs_per_batch: int, q_strides, k_strides, Lq: int, Lk: int, num_heads: int,
               head_dim: int, kv_lens=None, q_norm_w=None, k_norm_w=None, norm_eps: float = 1e-6, rope_cos=None,
               rope_sin=None, softmax_scale=None, q_norm_w2=None, k_norm_w2=None, norm_split: int = 0, impl: int = 0,
               rope_half: bool = False):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out"), (q_norm_w, "q_norm_w"), (k_norm_w, "k_norm_w")):
        _need(t, torch.bfloat16, n)
    _need(rope_cos, torch.float32, "rope_cos"); _need(rope_sin, torch.float32, "rope_sin"); _need(kv_lens, torch.int32, "kv_lens")
    if (q_norm_w is None) != (k_norm_w is None) or (rope_cos is None) != (rope_sin is None):
        raise OsbError("osb_attn_short: norm weights / rope tables must come in pairs")
    if (q_norm_w2 is None) != (k_norm_w2 is None) or (q_norm_w2 is not None and q_norm_w is None):
        raise OsbError("osb_attn_short: the second norm weight pair needs the first")
    H, D = num_heads, head_dim
    if D not in (64, 72, 128):
        raise OsbError(f"osb_attn_short failed (-1): head_dim {D} not built (64, 72, 128)")
    if rope_cos is not None and rope_half and D % 16:
        raise OsbError("osb_attn_short failed (-1): rotate-half RoPE needs head_dim % 16 == 0")
    dev = q.device
    s = torch.arange(num_seqs, device=dev)
    b, j = s // seqs_per_batch, s % seqs_per_batch

    def rows(strides, L):   # [num_seqs, L] row index of token t of sequence s
        bs, ss, ts = strides
        return (b * bs + j * ss)[:, None] + torch.arange(L, device=dev)[None] * ts

    rq, rk = rows(q_strides, Lq), rows(k_strides, Lk)
    qf = q[rq][..., : H * D].float().view(num_seqs, Lq, H, D).transpose(1, 2)      # [n, H, Lq, D]
    kf = k[rk][..., : H * D].float().view(num_seqs, Lk, H, D).transpose(1, 2)
    vf = v[rk][..., : H * D].float().view(num_seqs, Lk, H, D).transpose(1, 2)
    if q_norm_w is not None:
        def normed(x, w, w2, L):
            y = _rms(x, w.float(), norm_eps)
            if w2 is not None:
                y2 = _rms(x, w2.float(), norm_eps)
                sel = (torch.arange(L, device=dev) >= norm_split)[None, None, :, None]
                y = torch.where(sel, y2, y)
            return y
        qf, kf = normed(qf, q_norm_w, q_norm_w2, Lq), normed(kf, k_norm_w, k_norm_w2, Lk)
    if rope_cos is not None:
        rot = _rope_half if rope_half else _rope_interleaved
        qf, kf = rot(qf, rope_cos[:Lq], rope_sin[:Lq]), rot(kf, rope_cos[:Lk], rope_sin[:Lk])
    qf, kf = qf.to(torch.bfloat16).float(), kf.to(torch.bfloat16).float()        # staged operands are bf16
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    sc = (qf @ kf.transpose(-1, -2)) * scale
    if kv_lens is not None:
        dead = torch.arange(Lk, device=dev)[None, :] >= kv_lens.long()[:, None]
        sc = sc.masked_fill(dead[:, None, None, :], float("-inf"))
    m = sc.amax(-1, keepdim=True)
    p = torch.exp(sc - torch.where(torch.isinf(m), torch.zeros_like(m), m))
    l = p.sum(-1, keepdim=True)
    o = (p.to(torch.bfloat16).float() @ vf) / torch.where(l > 0, l, torch.ones_like(l))   # P is rounded before P V
    o = o.transpose(1, 2).reshape(num_seqs, Lq, H * D).to(torch.bfloat16)
    out[rq.reshape(-1), : H * D] = o.reshape(-1, H * D)
    _count("attn_short", (num_seqs, Lq, Lk, H, D))
    return out


# ---- causal 3D VAE ops (NDHWC) ---------------------------------------------------------------------------------
def group_stats(x, groups: int, eps: float = 1e-6):
    _need(x, torch.bfloat16, "x")
    assert x.dim() == 5 and x.is_contiguous()
    nb, C = x.shape[0], x.shape[-1]
    if groups <= 0 or C % groups or C % 8 or 256 % (C // 8) or groups > 1024:
        raise OsbError(f"osb_group_stats failed (-1): C/8 must divide 256 and groups C (C = {C}, groups {groups})")
    xf = x.float().reshape(nb, -1, groups, C // groups)
    mean = xf.mean(dim=(1, 3))
    var = (xf - mean[:, None, :, None]).pow(2).mean(dim=(1, 3))
    _count("group_stats", tuple(x.shape), launches=2)   # block partials + fp64 finalize
    return torch.stack((mean, torch.rsqrt(var + eps)), dim=-1)


def vae_prep(x, *, stats=None, gamma=None, beta=None, groups: int = 32, silu: bool = False, up=(1, 1, 1), pad=(0, 0, 0),
             cp=None, slack_bytes: int = 128):
    _need(x, torch.bfloat16, "x"); _need(stats, torch.float32, "stats"); _need(gamma, torch.bfloat16, "gamma")
    _need(beta, torch.bfloat16, "beta")
    assert x.dim() == 5 and x.is_contiguous()
    nb, T, H, W, C = x.shape
    cp = cp or C
    if C % 8 or cp % 8 or cp < C:
        raise OsbError(f"osb_vae_prep failed (-1): channels must be multiples of 8 (c {C} cp {cp})")
    if any(f not in (1, 2) for f in up):
        raise OsbError(f"osb_vae_prep failed (-1): upsample factors must be 1 or 2, got {tuple(up)}")
    if stats is not None and (gamma is None or beta is None or groups <= 0 or C % groups):
        raise OsbError("osb_vae_prep failed (-1): GroupNorm needs gamma, beta and a valid group count")
    y = x.float()
    if stats is not None:
        cg = C // groups
        mean = stats[..., 0].repeat_interleave(cg, dim=1)[:, None, None, None, :]
        rstd = stats[..., 1].repeat_interleave(cg, dim=1)[:, None, None, None, :]
        y = (y - mean) * rstd * gamma.float() + beta.float()
    if silu:
        y = y * torch.sigmoid(y)
    ft, fh, fw = up
    if ft > 1:   # first-frame rule: frame 0 once, every later frame ft times (T' = 1 + ft (T - 1))
        y = torch.cat((y[:, :1], y[:, 1:].repeat_interleave(ft, dim=1)), dim=1)
    if fh > 1:
        y = y.repeat_interleave(fh, dim=2)
    if fw > 1:
        y = y.repeat_interleave(fw, dim=3)
    pt, ph, pw = pad
    if pt or ph or pw:   # replicate: T at the front only (causal), H / W on both sides
        y = F.pad(y.permute(0, 4, 1, 2, 3), (pw, pw, ph, ph, pt, 0), mode="replicate").permute(0, 2, 3, 4, 1)
    if cp > C:
        y = F.pad(y, (0, cp - C))
    _count("vae_prep", (tuple(x.shape), up, pad))
    return y.to(torch.bfloat16).contiguous()


def pack_conv_weight(w, cp: int, narrow: bool, cout_pad=None):
    cout, cin, kt, kh, kw = w.shape
    co = cout_pad or cout
    if narrow:
        out = torch.zeros(co, kt * kh, 64, dtype=w.dtype, device=w.device)
        blk = torch.zeros(cout, kt * kh, kw, cp, dtype=w.dtype, device=w.device)
        blk[..., :cin] = w.permute(0, 2, 3, 4, 1).reshape(cout, kt * kh, kw, cin)
        out[:cout, :, : kw * cp] = blk.reshape(cout, kt * kh, kw * cp)
        return out.reshape(co, kt * kh * 64).to(torch.bfloat16).contiguous()
    out = torch.zeros(co, kt, kh, kw, cp, dtype=w.dtype, device=w.device)
    out[:cout, ..., :cin] = w.permute(0, 2, 3, 4, 1)
    return out.reshape(co, kt * kh * kw * cp).to(torch.bfloat16).contiguous()


def conv3d(x_pad, w_packed, bias, *, out_thw, stride=(1, 1, 1), taps=(3, 3, 3), narrow: bool = False, residual=None,
           block_n: int = 0):
    for t, n in ((x_pad, "x_pad"), (w_packed, "w_packed"), (bias, "bias"), (residual, "residual")):
        _need(t, torch.bfloat16, n)
    nb, tp, hp, wp, cp = x_pad.shape
    kt, kh, kw = taps
    cout = w_packed.shape[0]
    if any(s not in (1, 2) for s in stride):
        raise OsbError(f"osb_conv3d_ndhwc failed (-1): strides must be 1 or 2, got {tuple(stride)}")
    if any(k not in (1, 2, 3) for k in taps):
        raise OsbError(f"osb_conv3d_ndhwc failed (-1): taps must be 1..3, got {tuple(taps)}")
    if cout % 8:
        raise OsbError(f"osb_conv3d_ndhwc: Cout must be a multiple of 8 (pad the weights), got {cout}")
    if narrow:
        if cp not in (8, 16) or kw * cp > 64:
            raise OsbError("osb_conv3d_ndhwc: narrow mode needs Cp in {8,16} with kw*Cp <= 64")
        w = w_packed.float().view(cout, kt * kh, 64)[:, :, : kw * cp].reshape(cout, kt, kh, kw, cp)
    else:
        if cp % 64:
            raise OsbError(f"osb_conv3d_ndhwc: Cp must be a multiple of 64 (or use narrow mode), got {cp}")
        w = w_packed.float().view(cout, kt, kh, kw, cp)
    t_out, h_out, w_out = out_thw
    st, sh, sw = stride
    if (t_out - 1) * st + kt > tp or (h_out - 1) * sh + kh > hp or (w_out - 1) * sw + kw > wp:
        raise OsbError("osb_conv3d_ndhwc: padded input too small for the output")
    y = F.conv3d(x_pad.to(ACC_DTYPE).permute(0, 4, 1, 2, 3), w.to(ACC_DTYPE).permute(0, 4, 1, 2, 3), None, stride=stride)
    y = y[:, :, :t_out, :h_out, :w_out].permute(0, 2, 3, 4, 1)
    if bias is not None:
        y = y + bias.to(ACC_DTYPE)
    if residual is not None:
        y = y + residual.to(ACC_DTYPE)
    _count("conv3d", (tuple(x_pad.shape), cout, stride, narrow))
    return y.to(torch.bfloat16).contiguous()


def cfg_euler(cond, uncond, uncond2, x, *, g_txt: float, g_img: float = 1.0, g_img_map=None, dt: float, out=None):
    for t, n in ((cond, "cond"), (uncond, "uncond"), (uncond2, "uncond2"), (x, "x"), (g_img_map, "g_img_map")):
        _need(t, torch.bfloat16, n)
    if x.numel() % 8 or (g_img_map is not None and (g_img_map.numel() % 8 or x.numel() % g_img_map.numel())):
        raise OsbError("osb_cfg_euler failed (-1): element count and guidance map period must be multiples of 8, "
                       "the period dividing the count")
    c, u = cond.float(), uncond.float()
    if uncond2 is None:
        pred = u + g_txt * (c - u)
    else:
        u2 = uncond2.float()
        gi = g_img if g_img_map is None else g_img_map.float().reshape(-1).repeat(x.numel() // g_img_map.numel()).view_as(x)
        pred = u2 + gi * (u - u2) + g_txt * (c - u)
    y = (x.float() + dt * pred).to(torch.bfloat16)
    _count("cfg_euler", x.numel())
    if out is None:
        return y
    out.copy_(y)
    return out


# ---- head tiles (include/osb200.h osb_gemm_head_tiles / osb_attn_tiles): the double keeps the tile buffer as a dense
# [kinds, rows, heads*D] tensor - the byte layout of a tile is the kernels' business, the CONTRACT is which token row and
# head a value belongs to, what was applied to it (bias, RMSNorm, RoPE by position) and which keys a query may see. ------
# The tile map is host arithmetic of the binding itself (pure Python over a ctypes struct, no device needed): the double
# uses it as is, so the two can never disagree on how a sequence is tiled.
from osb200 import TileMap, tile_map  # noqa: E402,F401


class HeadTiles:
    def __init__(self, rows, tmap, kinds, heads, head_dim, device):
        if tmap.mode == 0:
            assert rows % tmap.L == 0, "rows must be whole sequences"
        else:
            assert tmap.T == tmap.L and tmap.S > 0 and rows % (tmap.S * tmap.T) == 0
        self.rows, self.map, self.kinds, self.heads, self.head_dim = rows, tmap, kinds, heads, head_dim
        self.dense = torch.zeros(kinds, rows, heads * head_dim, dtype=torch.bfloat16, device=device)


def _seq_pos(m, rows, device):
    r = torch.arange(rows, device=device)
    if m.mode == 0:
        return r // m.L, r % m.L
    b, rem = r // (m.T * m.S), r % (m.T * m.S)
    return b * m.S + rem % m.S, rem // m.S


def gemm_head_tiles(a, w, bias, tiles, *, nkinds, norm_w=(), rope=None, rope_kinds=0, eps=1e-6, kind0=0, general=False):
    for t, n in ((a, "a"), (w, "w"), (bias, "bias")):
        _need(t, torch.bfloat16, n)
    M, K = a.shape
    N = w.shape[0]
    H, D = tiles.heads, tiles.head_dim
    Cc = H * D
    assert M == tiles.rows and N % Cc == 0 and kind0 + N // Cc <= tiles.kinds and a.shape[1] == w.shape[1]
    if D not in (64, 72, 128) or H % 2:
        raise OsbError("osb_gemm_head_tiles failed (-1): head_dim / head count not built")
    if K % 8:
        raise OsbError(f"osb_gemm_head_tiles failed (-1): K must be a multiple of 8 (K {K})")
    if not 1 <= nkinds <= 4:
        raise OsbError(f"osb_gemm_head_tiles failed (-1): nkinds must be 1..4, got {nkinds}")
    if any(nw is not None for nw in norm_w[nkinds:]):
        raise OsbError("osb_gemm_head_tiles failed (-1): RMSNorm weight given for a kind >= nkinds")
    acc = a.float() @ w.float().t()
    if bias is not None:
        acc = acc + bias.float()
    _, pos = _seq_pos(tiles.map, M, a.device)
    for kidx in range(N // Cc):
        kind = kidx % nkinds
        x = acc[:, kidx * Cc:(kidx + 1) * Cc].reshape(M, H, D)
        nw = norm_w[kind] if kind < len(norm_w) else None
        if nw is not None:
            x = x * torch.rsqrt(x.pow(2).mean(-1, keepdim=True) + eps) * nw.float()
        if rope is not None and (rope_kinds >> kind) & 1:
            c, s_ = rope[0][pos][:, None, :], rope[1][pos][:, None, :]
            xa, xb = x[..., 0::2], x[..., 1::2]
            x = torch.stack((xa * c - xb * s_, xb * c + xa * s_), dim=-1).reshape(M, H, D)
        tiles.dense[kind0 + kidx] = x.reshape(M, Cc).to(torch.bfloat16)
    _count("gemm", (M, N, K, "head_tiles"))
    return tiles


def attn_tiles(q, kv, out, *, q_kind=0, k_kind=1, v_kind=2, Lk, num_seqs, kv_lens=None, softmax_scale=None,
               out_scatter=None, out_ld=None, out_map=None):
    H, D = q.heads, q.head_dim
    m = q.map
    if kv_lens is not None and m.G > 1:
        raise OsbError("attn_tiles: kv_lens applies to unpacked query maps only (G == 1); packed sequences see all Lk keys")
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    seq_q, pos_q = _seq_pos(m, q.rows, out.device)
    out_rows = None
    if out_map is not None:   # output rows in another token order: (seq, pos) -> row of `out`
        assert out_map.key()[4:] == m.key()[4:] and out_map.L == m.L
        so, po = _seq_pos(out_map, q.rows, out.device)
        inv = torch.empty(q.rows, dtype=torch.long, device=out.device)
        inv[so * m.L + po] = torch.arange(q.rows, device=out.device)
        out_rows = inv[seq_q * m.L + pos_q]
    seq_k, pos_k = _seq_pos(kv.map, kv.rows, out.device)
    assert int(seq_q.max()) + 1 == num_seqs
    for s in range(num_seqs):
        rq = (seq_q == s).nonzero().flatten()
        rk = (seq_k == s).nonzero().flatten()
        rk = rk[pos_k[rk].argsort()]
        n = Lk if kv_lens is None else min(int(kv_lens[s]), Lk)
        ro = rq if out_rows is None else out_rows[rq]
        if n <= 0:
            out[ro] = 0
            continue
        rk = rk[:n]
        qq = q.dense[q_kind][rq].float().view(-1, H, D).permute(1, 0, 2)
        kk = kv.dense[k_kind][rk].float().view(-1, H, D).permute(1, 0, 2)
        vv = kv.dense[v_kind][rk].float().view(-1, H, D).permute(1, 0, 2)
        sc = qq @ kk.transpose(-1, -2) * scale
        p = torch.exp(sc - sc.amax(-1, keepdim=True))
        # as the kernel: the UNnormalised P is rounded to bf16 for P V, the sum is taken over the unrounded P
        o = (p.to(torch.bfloat16).float() @ vv) / p.sum(-1, keepdim=True)
        out[ro] = o.permute(1, 0, 2).reshape(len(rq), H * D).to(torch.bfloat16)
    _count("attn_tiles", (num_seqs, m.L, Lk, H, D))
    return out
