"""MMDiT layers on the osb200 kernels — same classes, constructor arguments, state-dict keys and the same
block-`processor` plug-in hook as the reference's `opensora/models/mmdit/layers.py`
(`DoubleStreamBlock.set_processor / forward = self.processor(self, img, txt, vec, pe)` :295-306,
`SingleStreamBlock` :378-388).  The nn.Modules hold parameters; the two processor classes below ARE the drop-in:
they read the block's own parameters and run every FLOP on libosb200 (sm_90a):

  LN(no affine)+modulate -> `osb_ln_modulate`; every Linear -> `osb_gemm_bf16` (bias / GELU-tanh / gate*x+residual
  epilogues); QK-RMSNorm + RoPE + joint txt|img softmax attention -> `osb_attn_short` (per-stream norm weights via
  `norm_split`); `linear2(cat(attn, gelu(mlp)))` reads ONE [rows, 5C] buffer that the attention kernel and the
  GELU GEMM wrote side by side (no torch.cat materialisation, SURVEY.md §2.2 K9).

Any joint sequence length (the flash attention variant streams key blocks), both RoPE layouts (`EmbedND`
interleaved pairs and `LigerEmbedND` rotate-half) and both QKV checkpoint layouts (`fused_qkv` True / False)."""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
from torch import Tensor, nn

from .math import liger_rope, rope, rope_tables


def _osb():
    import osb200

    return osb200


class EmbedND(nn.Module):
    """layers.py:31-44."""

    def __init__(self, dim: int, theta: int, axes_dim: list[int]):
        super().__init__()
        self.dim, self.theta, self.axes_dim = dim, theta, axes_dim

    def forward(self, ids: Tensor) -> Tensor:
        emb = torch.cat([rope(ids[..., i], self.axes_dim[i], self.theta) for i in range(ids.shape[-1])], dim=-3)
        return emb.unsqueeze(1)


class LigerEmbedND(nn.Module):
    """layers.py:47-65."""

    def __init__(self, dim: int, theta: int, axes_dim: list[int]):
        super().__init__()
        self.dim, self.theta, self.axes_dim = dim, theta, axes_dim

    def forward(self, ids: Tensor):
        cs = [liger_rope(ids[..., i], self.axes_dim[i], self.theta) for i in range(ids.shape[-1])]
        cos = torch.cat([c for c, _ in cs], dim=-1).repeat(1, 1, 2).contiguous()
        sin = torch.cat([s for _, s in cs], dim=-1).repeat(1, 1, 2).contiguous()
        return (cos, sin)


def timestep_embedding(t: Tensor, dim, max_period=10000, time_factor: float = 1000.0):
    """layers.py:68-88 (the reference `torch.compile`s this; it is [B, 256] work once per step)."""
    t = time_factor * t
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(0, half, dtype=torch.float32) / half).to(t.device)
    args = t[:, None].float() * freqs[None]
    emb = torch.cat([torch.cos(args), torch.sin(args)], dim=-1)
    if dim % 2:
        emb = torch.cat([emb, torch.zeros_like(emb[:, :1])], dim=-1)
    if torch.is_floating_point(t):
        emb = emb.to(t)
    return emb


def _linear(x2d: Tensor, lin: nn.Linear, **kw) -> Tensor:
    return _osb().gemm(x2d, lin.weight, lin.bias, **kw)


class MLPEmbedder(nn.Module):
    def __init__(self, in_dim: int, hidden_dim: int):
        super().__init__()
        self.in_layer = nn.Linear(in_dim, hidden_dim, bias=True)
        self.silu = nn.SiLU()
        self.out_layer = nn.Linear(hidden_dim, hidden_dim, bias=True)

    def forward(self, x: Tensor) -> Tensor:
        h = _linear(x.to(self.in_layer.weight.dtype).contiguous(), self.in_layer)
        return _linear(torch.nn.functional.silu(h), self.out_layer)


class RMSNorm(nn.Module):
    """Parameter container (`scale`), layers.py:102-111; applied inside the attention kernel."""

    def __init__(self, dim: int):
        super().__init__()
        self.scale = nn.Parameter(torch.ones(dim))


class FusedRMSNorm(RMSNorm):
    pass


class QKNorm(nn.Module):
    def __init__(self, dim: int):
        super().__init__()
        self.query_norm = FusedRMSNorm(dim)
        self.key_norm = FusedRMSNorm(dim)


class SelfAttention(nn.Module):
    """Parameter container with the reference's attribute names (layers.py:138-152)."""

    def __init__(self, dim: int, num_heads: int = 8, qkv_bias: bool = False, fused_qkv: bool = True):
        super().__init__()
        self.num_heads, self.fused_qkv = num_heads, fused_qkv
        if fused_qkv:
            self.qkv = nn.Linear(dim, dim * 3, bias=qkv_bias)
        else:
            self.q_proj = nn.Linear(dim, dim, bias=qkv_bias)
            self.k_proj = nn.Linear(dim, dim, bias=qkv_bias)
            self.v_proj = nn.Linear(dim, dim, bias=qkv_bias)
        self.norm = QKNorm(dim // num_heads)
        self.proj = nn.Linear(dim, dim)


@dataclass
class ModulationOut:
    shift: Tensor
    scale: Tensor
    gate: Tensor


class Modulation(nn.Module):
    """Parameter container (layers.py:179-192); the processors read `lin` / `multiplier` and run the projection on
    osb200.  `forward` keeps the reference's return contract for callers outside the block path."""

    def __init__(self, dim: int, double: bool):
        super().__init__()
        self.is_double = double
        self.multiplier = 6 if double else 3
        self.lin = nn.Linear(dim, self.multiplier * dim, bias=True)

    def forward(self, vec: Tensor):
        out = _linear(torch.nn.functional.silu(vec).contiguous(), self.lin)[:, None, :].chunk(self.multiplier, dim=-1)
        return ModulationOut(*out[:3]), (ModulationOut(*out[3:]) if self.is_double else None)


def _check(x: Tensor):
    osb = _osb()
    osb.require_cuda_bf16(x, "MMDiT")
    return osb


def _rope(pe):
    """(cos, sin, rotate_half) for the attention kernel: EmbedND -> interleaved pairs, LigerEmbedND -> rotate-half.  The
    tables depend only on `pe`, which every block of a forward (and, with a cached `pe`, every step) shares: they are memoised on
    the tensor itself (57 slicing + contiguous passes per step otherwise)."""
    host = pe if isinstance(pe, Tensor) else pe[0]
    hit = getattr(host, "_osb_rope_tables", None)
    if hit is None or hit[0] != host._version:
        hit = (host._version, rope_tables(pe))
        try:
            host._osb_rope_tables = hit
        except Exception:   # a tensor subclass that refuses attributes: just recompute
            pass
    return hit[1]


# Sequence parallelism (Ulysses, the reference's `all_to_all` mode: opensora/models/mmdit/distributed.py:473-495): the joint
# txt|img sequence is split into P equal chunks; around attention q, k, v are exchanged "scatter heads / gather sequence" and
# the output back.  MMDiTModel sets the group for the duration of a forward; a processor running outside of it sees None.
_SP = {"group": None}


def _sp_group():
    return _SP["group"]


def _sp_attention(osb, qkv: Tensor, out_cols: int, B: int, Lloc: int, H: int, D: int, attn_kw: dict, norm_split_full: int,
                  dtype, device) -> Tensor:
    """softmax(q k^T) v over the FULL joint sequence from this rank's [B*Lloc, 3*H*D] q|k|v rows: heads are scattered and
    the sequence gathered with one all-to-all (q, k, v travel together), attention runs on H/P heads, and the output comes
    back with the inverse exchange.  Without a group it is the plain local attention."""
    import torch.distributed as dist

    from opensora.acceleration.communications import all_to_all

    g = _sp_group()
    P = dist.get_world_size(g) if g is not None else 1
    C = H * D
    if P == 1:
        ao = torch.empty(B * Lloc, out_cols, dtype=dtype, device=device)
        osb.attn_short(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ao[:, :C], num_seqs=B, seqs_per_batch=1,
                       q_strides=(Lloc, 0, 1), k_strides=(Lloc, 0, 1), Lq=Lloc, Lk=Lloc, num_heads=H, head_dim=D,
                       norm_split=norm_split_full, **attn_kw)
        return ao
    if H % P:
        raise ValueError(f"sequence parallel size {P} must divide the head count {H} (distributed.py:477-479)")
    Hp, L = H // P, Lloc * P
    full = all_to_all(qkv.view(B, Lloc, 3, H, D), g, scatter_dim=3, gather_dim=1).reshape(B * L, 3 * Hp * D)
    Cp = Hp * D
    ao_full = torch.empty(B * L, Cp, dtype=dtype, device=device)
    osb.attn_short(full[:, :Cp], full[:, Cp:2 * Cp], full[:, 2 * Cp:], ao_full, num_seqs=B, seqs_per_batch=1,
                   q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=Hp, head_dim=D,
                   norm_split=norm_split_full, **attn_kw)
    back = all_to_all(ao_full.view(B, L, Hp, D), g, scatter_dim=1, gather_dim=2).reshape(B * Lloc, C)
    if out_cols == C:
        return back
    ao = torch.empty(B * Lloc, out_cols, dtype=dtype, device=device)
    ao[:, :C] = back
    return ao


class _ProcessorBase:
    """What both processors share.  A processor holds NO model weights and touches only attributes the reference's own
    block classes have (`opensora/models/mmdit/layers.py:138-176,256-306,337-388`), so it can be installed with
    `block.set_processor(...)` on the reference's DoubleStreamBlock / SingleStreamBlock objects as well as on this
    package's.  Derived tensors (q|k|v weights concatenated for checkpoints with `fused_qkv=False`) are cached per
    block, keyed by the identity and version of the source parameters, so `.to()` / `load_state_dict` invalidate them."""

    def __init__(self):
        import weakref

        self._cache = weakref.WeakKeyDictionary()

    def _cached(self, block: nn.Module, name: str, sources, build):
        sig = tuple((t.data_ptr(), t._version, t.dtype, t.device) for t in sources if t is not None)
        ent = self._cache.setdefault(block, {})
        hit = ent.get(name)
        if hit is None or hit[0] != sig:
            ent[name] = hit = (sig, build())
        return hit[1]

    def _qkv(self, block: nn.Module, sa: nn.Module, name: str):
        """[3C, C] weight and [3C] bias in q|k|v row order for ONE GEMM, whichever way the checkpoint stores them."""
        if getattr(sa, "fused_qkv", hasattr(sa, "qkv")):
            return sa.qkv.weight, sa.qkv.bias
        ws = (sa.q_proj.weight, sa.k_proj.weight, sa.v_proj.weight)
        bs = (sa.q_proj.bias, sa.k_proj.bias, sa.v_proj.bias)
        return self._cached(block, name, ws + bs, lambda: (
            torch.cat(ws, 0).contiguous(), None if bs[0] is None else torch.cat(bs, 0).contiguous()))

    @staticmethod
    def _modulation(osb, mod: nn.Module, vec: Tensor):
        """layers.py:186-192 on osb200: lin(silu(vec)) -> fp32 [B, C] row views (row stride multiplier*C) the kernels take
        as shift / scale / gate.  When the model has already projected `vec` through EVERY block's modulation layer in one
        grouped GEMM (MMDiTModel.forward_ckpt: SURVEY.md 8f-2), the result rides on `vec` and this block takes its columns."""
        grouped = getattr(vec, "_osb_grouped_modulation", None)
        if grouped is not None and id(mod.lin) in grouped[1]:
            lo, hi = grouped[1][id(mod.lin)]
            out = grouped[0][:, lo:hi]
        else:
            out = osb.gemm(torch.nn.functional.silu(vec).contiguous(), mod.lin.weight, mod.lin.bias).float()
        mult = getattr(mod, "multiplier", None) or (mod.lin.out_features // mod.lin.in_features)
        c = out.chunk(mult, dim=-1)
        return ModulationOut(*c[:3]), (ModulationOut(*c[3:6]) if mult >= 6 else None)


class DoubleStreamBlockProcessor(_ProcessorBase):
    """osb200 implementation of layers.py:195-253 (and, under sequence parallelism, of distributed.py:473-495)."""

    def __call__(self, attn: nn.Module, img: Tensor, txt: Tensor, vec: Tensor, pe) -> tuple[Tensor, Tensor]:
        osb = _check(img)
        B, Li, C = img.shape
        Lt = txt.shape[1]            # may be 0 on a sequence-parallel rank whose chunk holds image tokens only
        L, H = Lt + Li, attn.num_heads
        D = C // H
        im1, im2 = self._modulation(osb, attn.img_mod, vec)
        tm1, tm2 = self._modulation(osb, attn.txt_mod, vec)
        img2, txt2 = img.reshape(B * Li, C).contiguous(), txt.reshape(B * Lt, C).contiguous()
        # q|k|v of both streams land in ONE joint [B*(Lt+Li), 3C] buffer in txt-then-img token order (layers.py:240-242)
        qkv = torch.empty(B * L, 3 * C, dtype=img.dtype, device=img.device)
        wi, bi = self._qkv(attn, attn.img_attn, "img_qkv")
        wt, bt = self._qkv(attn, attn.txt_attn, "txt_qkv")
        if Li:
            xi = osb.ln_modulate(img2, im1.shift, im1.scale, group_rows=Li)
        if Lt:
            xt = osb.ln_modulate(txt2, tm1.shift, tm1.scale, group_rows=Lt)
        for b in range(B):
            if Lt:
                osb.gemm(xt[b * Lt:(b + 1) * Lt], wt, bt, out=qkv[b * L:b * L + Lt])
            if Li:
                osb.gemm(xi[b * Li:(b + 1) * Li], wi, bi, out=qkv[b * L + Lt:(b + 1) * L])
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.txt_attn.norm.query_norm.scale, k_norm_w=attn.txt_attn.norm.key_norm.scale,
                  q_norm_w2=attn.img_attn.norm.query_norm.scale, k_norm_w2=attn.img_attn.norm.key_norm.scale,
                  rope_cos=cos, rope_sin=sin, rope_half=half)
        # tokens at joint position >= the FULL text length take the image stream's QK-norm weights
        split_full = getattr(vec, "_osb_txt_len", Lt)
        ao = _sp_attention(osb, qkv, C, B, L, H, D, kw, split_full, img.dtype, img.device)
        img_o, txt_o = torch.empty_like(img2), torch.empty_like(txt2)
        for b in range(B):  # x + gate * proj(attn)   (layers.py:247, 251)
            if Li:
                osb.gemm(ao[b * L + Lt:(b + 1) * L], attn.img_attn.proj.weight, attn.img_attn.proj.bias,
                         epilogue=osb.EPI_BIAS_GATE_RES, residual=img2[b * Li:(b + 1) * Li], gate=im1.gate[b:b + 1],
                         out=img_o[b * Li:(b + 1) * Li])
            if Lt:
                osb.gemm(ao[b * L:b * L + Lt], attn.txt_attn.proj.weight, attn.txt_attn.proj.bias,
                         epilogue=osb.EPI_BIAS_GATE_RES, residual=txt2[b * Lt:(b + 1) * Lt], gate=tm1.gate[b:b + 1],
                         out=txt_o[b * Lt:(b + 1) * Lt])
        # x + gate * MLP((1 + scale) * LN(x) + shift)   (layers.py:248, 252)
        for x_o, mod, mlp, n in ((img_o, im2, attn.img_mlp, Li), (txt_o, tm2, attn.txt_mlp, Lt)):
            if n == 0:
                continue
            xm = osb.ln_modulate(x_o, mod.shift, mod.scale, group_rows=n)
            hid = osb.gemm(xm, mlp[0].weight, mlp[0].bias, epilogue=osb.EPI_BIAS_GELU_TANH)
            osb.gemm(hid, mlp[2].weight, mlp[2].bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=x_o, gate=mod.gate,
                     group_rows=n, out=x_o)
        return img_o.view(B, Li, C), txt_o.view(B, Lt, C)


class DoubleStreamBlock(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, mlp_ratio: float, qkv_bias: bool = False, fused_qkv: bool = True):
        super().__init__()
        mlp_hidden_dim = int(hidden_size * mlp_ratio)
        self.num_heads, self.hidden_size, self.head_dim = num_heads, hidden_size, hidden_size // num_heads
        self.img_mod = Modulation(hidden_size, double=True)
        self.img_norm1 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.img_attn = SelfAttention(dim=hidden_size, num_heads=num_heads, qkv_bias=qkv_bias, fused_qkv=fused_qkv)
        self.img_norm2 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.img_mlp = nn.Sequential(nn.Linear(hidden_size, mlp_hidden_dim, bias=True), nn.GELU(approximate="tanh"),
                                     nn.Linear(mlp_hidden_dim, hidden_size, bias=True))
        self.txt_mod = Modulation(hidden_size, double=True)
        self.txt_norm1 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.txt_attn = SelfAttention(dim=hidden_size, num_heads=num_heads, qkv_bias=qkv_bias, fused_qkv=fused_qkv)
        self.txt_norm2 = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.txt_mlp = nn.Sequential(nn.Linear(hidden_size, mlp_hidden_dim, bias=True), nn.GELU(approximate="tanh"),
                                     nn.Linear(mlp_hidden_dim, hidden_size, bias=True))
        self.set_processor(DoubleStreamBlockProcessor())

    def set_processor(self, processor) -> None:
        self.processor = processor

    def get_processor(self):
        return self.processor

    def forward(self, img: Tensor, txt: Tensor, vec: Tensor, pe, **kwargs) -> tuple[Tensor, Tensor]:
        return self.processor(self, img, txt, vec, pe)


class SingleStreamBlockProcessor(_ProcessorBase):
    """osb200 implementation of layers.py:309-334."""

    def _split_weights(self, blk: nn.Module):
        """(W_qkv [3C,C], b_qkv, W_mlp [4C,C], b_mlp): row views of linear1, or packed from q_proj / k_proj / v_mlp."""
        C = blk.linear2.out_features
        if getattr(blk, "fused_qkv", hasattr(blk, "linear1")):
            w, b = blk.linear1.weight, blk.linear1.bias
            return w[:3 * C], b[:3 * C], w[3 * C:], b[3 * C:]
        src = (blk.q_proj.weight, blk.k_proj.weight, blk.v_mlp.weight, blk.q_proj.bias, blk.k_proj.bias, blk.v_mlp.bias)
        wq, bq = self._cached(blk, "qkv", src, lambda: (
            torch.cat([blk.q_proj.weight, blk.k_proj.weight, blk.v_mlp.weight[:C]], 0).contiguous(),
            torch.cat([blk.q_proj.bias, blk.k_proj.bias, blk.v_mlp.bias[:C]], 0).contiguous()))
        return wq, bq, blk.v_mlp.weight[C:], blk.v_mlp.bias[C:]

    def __call__(self, attn: nn.Module, x: Tensor, vec: Tensor, pe) -> Tensor:
        osb = _check(x)
        B, L, C = x.shape
        H = attn.num_heads
        D, M4 = C // H, attn.linear2.in_features - C
        mod, _ = self._modulation(osb, attn.modulation, vec)
        x2 = x.reshape(B * L, C).contiguous()
        xm = osb.ln_modulate(x2, mod.shift, mod.scale, group_rows=L)
        wq, bq, wm, bm = self._split_weights(attn)
        qkv = osb.gemm(xm, wq, bq)                                               # [B*L, 3C]
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.norm.query_norm.scale, k_norm_w=attn.norm.key_norm.scale, rope_cos=cos, rope_sin=sin,
                  rope_half=half)
        # [attn | gelu(mlp)] side by side: the attention output and the GELU GEMM write one [rows, C + 4C] buffer
        cat = _sp_attention(osb, qkv, C + M4, B, L, H, D, kw, 0, x.dtype, x.device)
        osb.gemm(xm, wm, bm, epilogue=osb.EPI_BIAS_GELU_TANH, out=cat[:, C:])
        out = osb.gemm(cat, attn.linear2.weight, attn.linear2.bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=x2,
                       gate=mod.gate, group_rows=L)
        return out.view(B, L, C)


class SingleStreamBlock(nn.Module):
    def __init__(self, hidden_size: int, num_heads: int, mlp_ratio: float = 4.0, qk_scale: float | None = None,
                 fused_qkv: bool = True):
        super().__init__()
        self.hidden_dim = self.hidden_size = hidden_size
        self.num_heads, self.head_dim = num_heads, hidden_size // num_heads
        self.scale = qk_scale or self.head_dim**-0.5
        self.fused_qkv = fused_qkv
        self.mlp_hidden_dim = int(hidden_size * mlp_ratio)
        if fused_qkv:
            self.linear1 = nn.Linear(hidden_size, hidden_size * 3 + self.mlp_hidden_dim)
        else:
            self.q_proj = nn.Linear(hidden_size, hidden_size)
            self.k_proj = nn.Linear(hidden_size, hidden_size)
            self.v_mlp = nn.Linear(hidden_size, hidden_size + self.mlp_hidden_dim)
        self.linear2 = nn.Linear(hidden_size + self.mlp_hidden_dim, hidden_size)
        self.norm = QKNorm(self.head_dim)
        self.pre_norm = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.mlp_act = nn.GELU(approximate="tanh")
        self.modulation = Modulation(hidden_size, double=False)
        self.set_processor(SingleStreamBlockProcessor())

    def set_processor(self, processor) -> None:
        self.processor = processor

    def get_processor(self):
        return self.processor

    def forward(self, x: Tensor, vec: Tensor, pe, **kwargs) -> Tensor:
        return self.processor(self, x, vec, pe)


class LastLayer(nn.Module):
    """layers.py:391-402."""

    def __init__(self, hidden_size: int, patch_size: int, out_channels: int):
        super().__init__()
        self.norm_final = nn.LayerNorm(hidden_size, elementwise_affine=False, eps=1e-6)
        self.linear = nn.Linear(hidden_size, patch_size * patch_size * out_channels, bias=True)
        self.adaLN_modulation = nn.Sequential(nn.SiLU(), nn.Linear(hidden_size, 2 * hidden_size, bias=True))

    def forward(self, x: Tensor, vec: Tensor) -> Tensor:
        osb = _check(x)
        B, L, C = x.shape
        m = _linear(torch.nn.functional.silu(vec).contiguous(), self.adaLN_modulation[1]).float()
        shift, scale = m.chunk(2, dim=1)
        xm = osb.ln_modulate(x.reshape(B * L, C).contiguous(), shift, scale, group_rows=L)
        return _linear(xm, self.linear).view(B, L, -1)
