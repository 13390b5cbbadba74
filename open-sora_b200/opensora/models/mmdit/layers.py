"""MMDiT layers on the osb200 kernels — same classes, constructor arguments, state-dict keys and the same
block-`processor` plug-in hook as the reference's `opensora/models/mmdit/layers.py`
(`DoubleStreamBlock.set_processor / forward = self.processor(self, img, txt, vec, pe)` :295-306,
`SingleStreamBlock` :378-388).  The nn.Modules hold parameters; the two processor classes below ARE the drop-in:
they read the block's own parameters and run every FLOP on libosb200 (sm_90a).  Any joint sequence length (the
flash attention variant streams key blocks), both RoPE layouts (`EmbedND` interleaved pairs and `LigerEmbedND`
rotate-half) and both QKV checkpoint layouts (`fused_qkv` True / False).

A block runs four stages: LN(no affine)+modulate, the q|k|v GEMM, joint txt|img attention followed by `proj`, and the
MLP.  A single block has no `proj`: its q|k|v and mlp GEMMs are the rows of linear1, and `linear2(cat(attn, gelu(mlp)))`
reads ONE [rows, C + M] buffer that the attention and the GELU GEMM write side by side (no torch.cat, SURVEY.md §2.2 K9).

`block_gemms` is the one description of which rows of which Linears make up each GEMM of a block.  The bf16 weights
(views, or a cached concatenation), the e4m3 weights (`Fp8State.weight`), the LoRA / DoRA packs (its slices are
`lora_pack` groups) and the model's `fp8_mlp_linears()` / `fp8_proj_linears()` derive from it.

Each processor picks once, per stage, the format of the activation that stage's GEMM reads: a bf16 tensor, or e4m3
codes with fp32 scales (one per row, or per 1 x 128 block) in workspaces of the model's `Fp8State`.  It then runs one
sequence of stages, and the helpers dispatch on the format:
  `_ln`         `osb_ln_modulate`, or `osb_ln_modulate_fp8` (one scale per row);
  `_gemm`       `osb_gemm_bf16`, or `osb_gemm_fp8_blocks` on e4m3 weights with per-output-channel scales; bias,
                GELU-tanh (bf16 or block-scaled e4m3 out) and gate * x + residual epilogues; with an adapter
                `osb_gemm_lora` / `osb_gemm_fp8_lora` (the unmerged update U (s B)^T, and DoRA's column scale, in the
                same fp32 accumulator);
  `_adapters`   the Linears whose GEMMs read one input share one pack and one down projection U = x A_cat^T (`_down`):
                a bf16 GEMM, or an FP8 GEMM on the codes the base GEMM reads with A_cat quantized per row;
  `_attention`  QK-RMSNorm + RoPE + softmax attention (`osb_attn_short`, or `osb_attn_fp8`), writing bf16 or e4m3
                with block scales, locally or through the Ulysses exchange.

Which stages read e4m3:
  default                       none.  LoRA / DoRA (opensora/utils/lora.py) run on the bf16 GEMMs; without an adapter
                                the launches are those of the plain model.
  MMDiTModel.enable_fp8()       the MLPs: fc1 (its GELU epilogue emits the block-scaled codes fc2 reads) and fc2; a
                                single block's mlp rows, on their own FP8 LN pass, and linear2, whose attention half
                                `osb_quant_blocks_fp8` fills from the bf16 attention output.
  ... projections=True          every block GEMM: q|k|v on per-row codes, `proj` / linear2 on the attention output as
                                block-scaled codes, written by `osb_attn_fp8_blocks` itself when FP8 attention is on;
                                a single block's q|k|v and mlp GEMMs read ONE FP8 LN pass.
  ... lora=True                 adapters on the e4m3 GEMMs run on them instead of being refused.
  enable_fp8_attention()        none: only the attention kernel changes (`osb_attn_fp8`).
The model hands its FP8 state to the processors on `vec` (`_osb_fp8`, an `Fp8State`; `_osb_fp8_attn`, an
`Fp8AttnState`)."""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch
from torch import Tensor, nn

from opensora.utils.lora import adapters_of, lora_pack

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


def linear_parts(lin: nn.Module, k_pad: int = 0):
    """(weight, bias, lora) of a Linear the forward sends to osb200: lora is None, or (A_cat [R, K + k_pad], B_cat,
    DoRA column scale or None) of its active adapters (lora_pack)."""
    if not adapters_of(lin):
        return lin.weight, lin.bias, None
    A, (B,), (S,) = lora_pack([[(lin, 0, lin.out_features)]], k_pad)
    return lin.weight, lin.bias, (A, B, S)


def _gemm(osb, x, w, b, lora=None, u: Tensor | None = None, **kw):
    """epilogue(x W^T + b) on the kernel of the input's format: a bf16 x (w bf16) runs `gemm`; an e4m3
    x = (codes, scales) (w = (codes, per-output-channel scales)) runs `gemm_fp8_blocks`.  With lora = (A_cat, B,
    col_scale) and its down projection u = x A_cat^T (`_down`), the unmerged update u B^T (times DoRA's column scale)
    joins the same accumulator: `gemm_lora` / `gemm_fp8_lora`.  A B of None (a pack group without an adapted Linear)
    adds nothing."""
    fp8 = not isinstance(x, Tensor)
    if lora is None or lora[1] is None:
        return osb.gemm_fp8_blocks(*x, *w, b, **kw) if fp8 else osb.gemm(x, w, b, **kw)
    if lora[2] is not None:
        kw["col_scale"] = lora[2]
    return osb.gemm_fp8_lora(*x, *w, b, u, lora[1], **kw) if fp8 else osb.gemm_lora(x, w, b, u, lora[1], **kw)


def _down(osb, x, lora, fp8: Fp8State | None = None, key=None) -> Tensor | None:
    """U = x A_cat^T of the adapters `lora` (a lora_pack result or one group of it, A_cat first; None without
    adapters): a bf16 `gemm`, or on e4m3 x = (codes, scales) `Fp8State.down` (A_cat quantized once per `key`)."""
    if lora is None:
        return None
    if isinstance(x, Tensor):
        return osb.gemm(x, lora[0])
    return fp8.down(osb, key, lora[0], *x)


def _linear(x2d: Tensor, lin: nn.Linear, **kw) -> Tensor:
    osb = _osb()
    w, b, lora = linear_parts(lin)
    return _gemm(osb, x2d, w, b, lora, _down(osb, x2d, lora), **kw)


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


class Fp8AttnState:
    """What the FP8 attention path of one MMDiTModel keeps: the workspaces of `osb200.attn_fp8`, one per (B, L, heads,
    device), reused by every block."""

    def __init__(self):
        self._ws = {}

    def workspace(self, osb, B: int, L: int, H: int, device):
        key = (B, L, H, device)
        ws = self._ws.get(key)
        if ws is None:
            ws = self._ws[key] = osb.attn_fp8_workspace(B, L, H, device)
        return ws


def _attention(osb, vec: Tensor, qkv: Tensor, out, B: int, L: int, H: int, attn_kw: dict, norm_split: int) -> None:
    """Joint self-attention of this rank's [B*L, 3C] q|k|v rows (B sequences of L tokens, H heads) into `out`: bf16
    [B*L, C] columns, or the e4m3 (codes, 1 x 128 block scales) input of the GEMM that reads it.

    The kernel is `osb_attn_short`, or `osb_attn_fp8` with FP8 attention on (`vec._osb_fp8_attn`).  An e4m3 `out` is
    the bf16 output quantized by `osb_quant_blocks_fp8`, except with FP8 attention and FP8 projections both on: then
    `osb_attn_fp8_blocks` writes the codes and the per-(token, head) scales itself.  The two differ in bits, and FP8
    MLPs alone keep the bf16 output of `enable_fp8_attention()` in front of their quantizer.

    Under sequence parallelism (Ulysses) one all-to-all scatters the heads and gathers the sequence (q, k, v travel
    together), the kernel runs on H/P heads of the full sequence, and the inverse exchange brings each output tensor
    back as bytes (bf16 rows, or codes and scales).  A (token, head) block is quantized alone either way, so the codes
    equal the single-rank ones."""
    import torch.distributed as dist

    from opensora.acceleration.communications import all_to_all

    fa, fp8 = getattr(vec, "_osb_fp8_attn", None), getattr(vec, "_osb_fp8", None)
    dst = out
    if not isinstance(out, Tensor) and (fa is None or not fp8.proj):
        dst = torch.empty(out[0].shape, dtype=qkv.dtype, device=qkv.device)
    D = qkv.shape[1] // (3 * H)

    def run(src: Tensor, o, Ls: int, Hs: int) -> None:
        C = Hs * D
        q, k, v = src[:, :C], src[:, C:2 * C], src[:, 2 * C:]
        kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(Ls, 0, 1), k_strides=(Ls, 0, 1), Lq=Ls, Lk=Ls, num_heads=Hs,
                  head_dim=D, norm_split=norm_split, **attn_kw)
        if fa is None:
            osb.attn_short(q, k, v, o, **kw)
        elif isinstance(o, Tensor):
            osb.attn_fp8(q, k, v, o, workspace=fa.workspace(osb, B, Ls, Hs, src.device), **kw)
        else:
            osb.attn_fp8_blocks(q, k, v, *o, workspace=fa.workspace(osb, B, Ls, Hs, src.device), **kw)

    g = _sp_group()
    P = dist.get_world_size(g) if g is not None else 1
    if P == 1:
        run(qkv, dst, L, H)
    else:
        if H % P:
            raise ValueError(f"sequence parallel size {P} must divide the head count {H} (distributed.py:477-479)")
        full = all_to_all(qkv.view(B, L, 3, H, D), g, scatter_dim=3, gather_dim=1).reshape(B * L * P, -1)
        parts = [dst] if isinstance(dst, Tensor) else list(dst)
        res = [torch.empty(B * L * P, t.shape[1] // P, dtype=t.dtype, device=t.device) for t in parts]
        run(full, res[0] if isinstance(dst, Tensor) else tuple(res), L * P, H // P)
        for t, r in zip(parts, res):
            back = all_to_all(r.view(torch.uint8).view(B, L * P, H // P, -1), g, scatter_dim=1, gather_dim=2)
            t.copy_(back.view(t.dtype).reshape(B * L, -1))
    if dst is not out:
        osb.quant_blocks_fp8(dst, out=out[0], out_scale=out[1])


# The GEMMs that run on e4m3 only with enable_fp8(projections=True); the other block GEMMs do with any enable_fp8().
PROJ_GEMMS = ("qkv", "proj")


def block_gemms(blk: nn.Module, kind: str) -> dict:
    """The GEMMs of one stream of a block: kind "img" / "txt" of a double block (`qkv`, `proj`, `fc1`, `fc2`) or
    "single" (`qkv`, `mlp`, `linear2`), each as the (linear, row_lo, row_hi) slices its output rows are made of, in
    order (the group format of `lora_pack`).  q|k|v is one GEMM whichever way the checkpoint stores it (`fused_qkv`);
    a single block's linear1 (or v_mlp) holds its q|k|v (or v) rows first and the mlp rows after them."""
    def whole(lin):
        return lin, 0, lin.out_features

    if kind == "single":
        C = blk.linear2.out_features
        if getattr(blk, "fused_qkv", hasattr(blk, "linear1")):
            l1, lo = blk.linear1, 3 * C
            qkv = [(l1, 0, lo)]
        else:
            l1, lo = blk.v_mlp, C
            qkv = [whole(blk.q_proj), whole(blk.k_proj), (l1, 0, lo)]
        return {"qkv": qkv, "mlp": [(l1, lo, l1.out_features)], "linear2": [whole(blk.linear2)]}
    sa, mlp = (blk.img_attn, blk.img_mlp) if kind == "img" else (blk.txt_attn, blk.txt_mlp)
    qkv = (sa.qkv,) if getattr(sa, "fused_qkv", hasattr(sa, "qkv")) else (sa.q_proj, sa.k_proj, sa.v_proj)
    return {"qkv": [whole(lin) for lin in qkv], "proj": [whole(sa.proj)], "fc1": [whole(mlp[0])], "fc2": [whole(mlp[2])]}


def _rows(slices):
    """(weight, bias) of a GEMM given by its block_gemms slices: row views of one Linear, or the rows concatenated."""
    if len(slices) == 1:
        lin, lo, hi = slices[0]
        return lin.weight[lo:hi], None if lin.bias is None else lin.bias[lo:hi]
    w = torch.cat([lin.weight[lo:hi] for lin, lo, hi in slices])
    return w, None if slices[0][0].bias is None else torch.cat([lin.bias[lo:hi] for lin, lo, hi in slices])


class Fp8State:
    """What the FP8 path of one MMDiTModel keeps: the e4m3 copy of every block GEMM that runs on FP8, quantized per
    output channel (`weight`); e4m3 / scale workspaces reused by every block, one per name and shape (`buf`); and,
    with `lora`, the e4m3 copy of each adapter pack's A_cat (`down`).  With `proj` the q|k|v and attention-output GEMMs
    run on FP8 too (PROJ_GEMMS)."""

    def __init__(self, proj: bool = False, lora: bool = False):
        self.proj, self.lora = proj, lora
        self._w, self._ws, self._la = {}, {}, {}

    def weight(self, osb, blk: nn.Module, kind: str, name: str, slices):
        """((e4m3 codes, per-output-channel scales), bias) of GEMM `name` of block_gemms(blk, kind) = `slices`,
        quantized once."""
        key = (id(blk), kind, name)
        hit = self._w.get(key)
        if hit is None or hit[0] is not blk:
            if not self.lora and any(adapters_of(lin) for lin, _, _ in slices):
                what, lin = ("FP8 projections", "a projection") if name in PROJ_GEMMS else ("FP8 MLPs", "an MLP")
                raise ValueError(f"{what}: a LoRA / DoRA adapter on {lin} Linear cannot run on the FP8 path; "
                                 "unload_lora or disable_fp8 first")
            w, b = _rows(slices)
            q, s = osb.quant_blocks_fp8(w, block=w.shape[1])
            hit = self._w[key] = (blk, ((q, s.view(-1)), b))
        return hit[1]

    def down(self, osb, key, A: Tensor, a8: Tensor, a_s: Tensor) -> Tensor:
        """U = x A^T (bf16 [rows, R]) of the adapters whose GEMMs read the e4m3 input (a8, a_s), on the block-scaled FP8
        GEMM.  A (a pack's A_cat) is quantized per row once per `key` and A: lora_pack hands out a new A_cat whenever
        the adapter state changes (reload, edited A / B, DoRA magnitude or base weight)."""
        hit = self._la.get(key)
        if hit is None or hit[0] is not A:
            q, sc = osb.quant_blocks_fp8(A, block=A.shape[1])
            hit = self._la[key] = (A, q, sc.view(-1))
        return osb.gemm_fp8_blocks(a8, a_s, hit[1], hit[2])

    def buf(self, name: str, *shape, dtype=torch.float32, device=None) -> Tensor:
        key = (name, shape, dtype, device)
        t = self._ws.get(key)
        if t is None:
            t = self._ws[key] = torch.empty(shape, dtype=dtype, device=device)
        return t


# Activations between the stages of a block are in the format of the GEMM that reads them, which the processor picks
# per stage: a bf16 tensor (fp8 None), or e4m3 (codes, fp32 scales) in workspaces of the model's Fp8State.
def _ln(osb, fp8: Fp8State | None, x: Tensor, mod, n: int, name: str):
    """(1 + scale) * LN(x) + shift per sample of n rows: bf16 (`osb_ln_modulate`), or with fp8 e4m3 codes with one
    scale per row (`osb_ln_modulate_fp8`) in workspace `name`."""
    if fp8 is None:
        return osb.ln_modulate(x, mod.shift, mod.scale, group_rows=n)
    rows, C = x.shape
    return osb.ln_modulate_fp8(x, mod.shift, mod.scale, group_rows=n,
                               out=fp8.buf(name, rows, C, dtype=torch.float8_e4m3fn, device=x.device),
                               out_scale=fp8.buf(name + ".s", rows, device=x.device))


def _act(fp8: Fp8State | None, name: str, rows: int, cols: int, device):
    """An empty [rows, cols] activation: bf16, or with fp8 e4m3 codes with 1 x 128 block scales (workspace `name`)."""
    if fp8 is None:
        return torch.empty(rows, cols, dtype=torch.bfloat16, device=device)
    return (fp8.buf(name, rows, cols, dtype=torch.float8_e4m3fn, device=device),
            fp8.buf(name + ".s", rows, cols // 128, device=device))


def _take(x, rows: slice):
    """Rows of an activation; None stays None."""
    if x is None:
        return None
    return x[rows] if isinstance(x, Tensor) else (x[0][rows], x[1][rows])


def _cols(x, lo: int, hi: int):
    """Columns lo..hi of an activation (of an e4m3 one with their block scales; lo, hi multiples of 128)."""
    return x[:, lo:hi] if isinstance(x, Tensor) else (x[0][:, lo:hi], x[1][:, lo // 128:hi // 128])


def _gelu_into(osb, out) -> dict:
    """Epilogue arguments of a GEMM that writes GELU-tanh into the activation `out`."""
    if isinstance(out, Tensor):
        return dict(epilogue=osb.EPI_BIAS_GELU_TANH, out=out)
    return dict(epilogue=osb.EPI_BIAS_GELU_TANH_FP8, out=out[0], out_scale=out[1])


def _adapters(osb, fp8: Fp8State | None, x, key, groups):
    """The adapters of the GEMMs `groups` (block_gemms slices) that all read x, as ONE lora_pack with ONE down projection
    (`_down`): ([(A_cat, B, col_scale) per group], U), or ([None] * len(groups), None) without an adapter.  On e4m3
    input they run only with enable_fp8(lora=True)."""
    p = None if fp8 is not None and not fp8.lora else lora_pack(groups)
    if p is None:
        return [None] * len(groups), None
    return [(p[0], B, S) for B, S in zip(p[1], p[2])], _down(osb, x, p, fp8, key)


class _ProcessorBase:
    """What both processors share.  A processor holds NO model weights and touches only attributes the reference's own
    block classes have (`opensora/models/mmdit/layers.py:138-176,256-306,337-388`), so it can be installed with
    `block.set_processor(...)` on the reference's DoubleStreamBlock / SingleStreamBlock objects as well as on this
    package's.  Weights of a GEMM made of several Linears (q|k|v of checkpoints with `fused_qkv=False`) are concatenated
    once and cached per block, keyed by the identity and version of the source parameters, so `.to()` /
    `load_state_dict` invalidate them."""

    def __init__(self):
        import weakref

        self._cache = weakref.WeakKeyDictionary()

    def _cached(self, block: nn.Module, name, sources, build):
        sig = tuple((t.data_ptr(), t._version, t.dtype, t.device) for t in sources if t is not None)
        ent = self._cache.setdefault(block, {})
        hit = ent.get(name)
        if hit is None or hit[0] != sig:
            ent[name] = hit = (sig, build())
        return hit[1]

    def _weight(self, osb, blk: nn.Module, kind: str, gemms: dict, name: str, fp8: Fp8State | None):
        """(weight, bias) of GEMM `name` of gemms = block_gemms(blk, kind): bf16, or with fp8 its e4m3 copy."""
        slices = gemms[name]
        if fp8 is not None:
            return fp8.weight(osb, blk, kind, name, slices)
        if len(slices) == 1:
            return _rows(slices)
        return self._cached(blk, (kind, name), [t for lin, _, _ in slices for t in (lin.weight, lin.bias)],
                            lambda: _rows(slices))

    @staticmethod
    def _modulation(mod: nn.Module, vec: Tensor):
        """layers.py:186-192 on osb200: lin(silu(vec)) -> fp32 [B, C] row views (row stride multiplier*C) the kernels take
        as shift / scale / gate.  When the model has already projected `vec` through EVERY block's modulation layer in one
        grouped GEMM (MMDiTModel.forward_ckpt: SURVEY.md 8f-2), the result rides on `vec` and this block takes its columns."""
        grouped = getattr(vec, "_osb_grouped_modulation", None)
        if grouped is not None and id(mod.lin) in grouped[1]:
            lo, hi = grouped[1][id(mod.lin)]
            out = grouped[0][:, lo:hi]
        else:
            out = _linear(torch.nn.functional.silu(vec).contiguous(), mod.lin).float()
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
        fp8 = getattr(vec, "_osb_fp8", None)                 # the MLPs read e4m3 with FP8 on
        p8 = fp8 if fp8 is not None and fp8.proj else None   # q|k|v and proj only with FP8 projections
        im1, im2 = self._modulation(attn.img_mod, vec)
        tm1, tm2 = self._modulation(attn.txt_mod, vec)
        img2, txt2 = img.reshape(B * Li, C).contiguous(), txt.reshape(B * Lt, C).contiguous()
        img_o, txt_o = torch.empty_like(img2), torch.empty_like(txt2)
        # per stream: input and output rows, both modulations, tokens per sample, first position in the joint txt|img
        # sequence (layers.py:240-242), GEMMs
        streams = (("img", img2, img_o, im1, im2, Li, Lt, block_gemms(attn, "img")),
                   ("txt", txt2, txt_o, tm1, tm2, Lt, 0, block_gemms(attn, "txt")))
        # q|k|v of both streams land in ONE joint [B*(Lt+Li), 3C] buffer; an adapter's down projection runs once over
        # all rows of a stream.  Each stream has its own LN workspace: both are read after both are written.
        qkv = torch.empty(B * L, 3 * C, dtype=img.dtype, device=img.device)
        ins = []
        for kind, x2, _, m1, _, n, off, g in streams:
            if n:
                xq = _ln(osb, p8, x2, m1, n, "x." + kind)
                (lq,), u = _adapters(osb, p8, xq, (id(attn), kind, "qkv"), [g["qkv"]])
                ins.append((xq, self._weight(osb, attn, kind, g, "qkv", p8), lq, u, n, off))
        for b in range(B):
            for xq, (w, bias), lq, u, n, off in reversed(ins):   # txt rows first
                r = slice(b * n, (b + 1) * n)
                _gemm(osb, _take(xq, r), w, bias, lq, _take(u, r), out=qkv[b * L + off:b * L + off + n])
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.txt_attn.norm.query_norm.scale, k_norm_w=attn.txt_attn.norm.key_norm.scale,
                  q_norm_w2=attn.img_attn.norm.query_norm.scale, k_norm_w2=attn.img_attn.norm.key_norm.scale,
                  rope_cos=cos, rope_sin=sin, rope_half=half)
        ao = _act(p8, "ao", B * L, C, img.device)
        # tokens at joint position >= the FULL text length take the image stream's QK-norm weights
        _attention(osb, vec, qkv, ao, B, L, H, kw, getattr(vec, "_osb_txt_len", Lt))
        # x + gate * proj(attn)   (layers.py:247, 251); both output projections read `ao`: one down projection
        lps, up = _adapters(osb, p8, ao, (id(attn), "proj"), [g["proj"] for *_, g in streams])
        wps = [self._weight(osb, attn, kind, g, "proj", p8) for kind, *_, g in streams]
        for b in range(B):
            for (_, x2, x_o, m1, _, n, off, _), (w, bias), lp in zip(streams, wps, lps):
                if n:
                    jr, sr = slice(b * L + off, b * L + off + n), slice(b * n, (b + 1) * n)
                    _gemm(osb, _take(ao, jr), w, bias, lp, _take(up, jr), epilogue=osb.EPI_BIAS_GATE_RES,
                          residual=x2[sr], gate=m1.gate[b:b + 1], out=x_o[sr])
        # x + gate * MLP((1 + scale) * LN(x) + shift)   (layers.py:248, 252)
        for kind, _, x_o, _, m2, n, _, g in streams:
            if n:
                xm = _ln(osb, fp8, x_o, m2, n, "x." + kind)
                (l1,), u1 = _adapters(osb, fp8, xm, (id(attn), kind, "fc1"), [g["fc1"]])
                h = _act(fp8, "h", x_o.shape[0], sum(hi - lo for _, lo, hi in g["fc1"]), img.device)
                _gemm(osb, xm, *self._weight(osb, attn, kind, g, "fc1", fp8), l1, u1, **_gelu_into(osb, h))
                (l2,), u2 = _adapters(osb, fp8, h, (id(attn), kind, "fc2"), [g["fc2"]])
                _gemm(osb, h, *self._weight(osb, attn, kind, g, "fc2", fp8), l2, u2, epilogue=osb.EPI_BIAS_GATE_RES,
                      residual=x_o, gate=m2.gate, group_rows=n, out=x_o)
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

    def __call__(self, attn: nn.Module, x: Tensor, vec: Tensor, pe) -> Tensor:
        osb = _check(x)
        B, L, C = x.shape
        H = attn.num_heads
        M = attn.linear2.in_features - C
        fp8 = getattr(vec, "_osb_fp8", None)                 # mlp and linear2 read e4m3 with FP8 on
        p8 = fp8 if fp8 is not None and fp8.proj else None   # qkv only with FP8 projections
        mod, _ = self._modulation(attn.modulation, vec)
        x2 = x.reshape(B * L, C).contiguous()
        g = block_gemms(attn, "single")
        xq = _ln(osb, p8, x2, mod, L, "x.single")
        if p8 is fp8:   # qkv and mlp read ONE LN+modulate output, with one down projection for their adapters
            (lq, lm), uq = _adapters(osb, p8, xq, (id(attn), "linear1"), [g["qkv"], g["mlp"]])
            xm, um = xq, uq
        else:           # FP8 MLPs alone: q|k|v on the bf16 LN output, the mlp part on its own FP8 LN pass
            (lq,), uq = _adapters(osb, p8, xq, None, [g["qkv"]])
            xm = _ln(osb, fp8, x2, mod, L, "x.single")
            (lm,), um = _adapters(osb, fp8, xm, (id(attn), "mlp"), [g["mlp"]])
        qkv = _gemm(osb, xq, *self._weight(osb, attn, "single", g, "qkv", p8), lq, uq)   # [B*L, 3C]
        cos, sin, half = _rope(pe)
        kw = dict(q_norm_w=attn.norm.query_norm.scale, k_norm_w=attn.norm.key_norm.scale, rope_cos=cos, rope_sin=sin,
                  rope_half=half)
        # [attn | gelu(mlp)] side by side: the attention and the GELU GEMM write ONE [rows, C + M] buffer that linear2
        # reads (no torch.cat)
        cat = _act(fp8, "cat", B * L, C + M, x.device)
        _attention(osb, vec, qkv, _cols(cat, 0, C), B, L, H, kw, 0)
        _gemm(osb, xm, *self._weight(osb, attn, "single", g, "mlp", fp8), lm, um,
              **_gelu_into(osb, _cols(cat, C, C + M)))
        (l2,), u2 = _adapters(osb, fp8, cat, (id(attn), "linear2"), [g["linear2"]])
        out = _gemm(osb, cat, *self._weight(osb, attn, "single", g, "linear2", fp8), l2, u2,
                    epilogue=osb.EPI_BIAS_GATE_RES, residual=x2, gate=mod.gate, group_rows=L)
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
