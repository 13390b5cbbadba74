"""MMDiTModel / `Flux` factory with the reference's constructor, registry key ("flux"), forward signature and
state-dict keys (`opensora/models/mmdit/model.py:38-303`), running on the osb200 kernels.  Forward-only:
`grad_ckpt_settings` is accepted and ignored (activation checkpointing is training-only, SURVEY.md §2 #9)."""
from __future__ import annotations

from dataclasses import dataclass

import torch
from torch import Tensor, nn

from opensora.registry import MODELS

from opensora.utils.lora import adapters_of, lora_pack

from .layers import (PROJ_GEMMS, DoubleStreamBlock, EmbedND, Fp8AttnState, Fp8State, LastLayer, LigerEmbedND,
                     MLPEmbedder, SingleStreamBlock, _down, _gemm, block_gemms, linear_parts, timestep_embedding)


@dataclass
class MMDiTConfig:
    model_type = "MMDiT"
    from_pretrained: str
    cache_dir: str
    in_channels: int
    vec_in_dim: int
    context_in_dim: int
    hidden_size: int
    mlp_ratio: float
    num_heads: int
    depth: int
    depth_single_blocks: int
    axes_dim: list
    theta: int
    qkv_bias: bool
    guidance_embed: bool
    cond_embed: bool = False
    fused_qkv: bool = True
    grad_ckpt_settings: tuple | None = None
    use_liger_rope: bool = False
    patch_size: int = 2

    def get(self, attribute_name, default=None):
        return getattr(self, attribute_name, default)

    def __contains__(self, attribute_name):
        return hasattr(self, attribute_name)


class MMDiTModel(nn.Module):
    config_class = MMDiTConfig

    def __init__(self, config: MMDiTConfig):
        super().__init__()
        self.config = config
        self.in_channels = self.out_channels = config.in_channels
        self.patch_size = config.patch_size
        if config.hidden_size % config.num_heads != 0:
            raise ValueError(f"Hidden size {config.hidden_size} must be divisible by num_heads {config.num_heads}")
        pe_dim = config.hidden_size // config.num_heads
        if sum(config.axes_dim) != pe_dim:
            raise ValueError(f"Got {config.axes_dim} but expected positional dim {pe_dim}")
        self.hidden_size, self.num_heads = config.hidden_size, config.num_heads
        self.pe_embedder = (LigerEmbedND if config.use_liger_rope else EmbedND)(dim=pe_dim, theta=config.theta,
                                                                                 axes_dim=config.axes_dim)
        self.img_in = nn.Linear(self.in_channels, self.hidden_size, bias=True)
        self.time_in = MLPEmbedder(in_dim=256, hidden_dim=self.hidden_size)
        self.vector_in = MLPEmbedder(config.vec_in_dim, self.hidden_size)
        self.guidance_in = MLPEmbedder(in_dim=256, hidden_dim=self.hidden_size) if config.guidance_embed else nn.Identity()
        self.cond_in = nn.Linear(self.in_channels + self.patch_size**2, self.hidden_size, bias=True) \
            if config.cond_embed else nn.Identity()
        self.txt_in = nn.Linear(config.context_in_dim, self.hidden_size)
        self.double_blocks = nn.ModuleList([
            DoubleStreamBlock(self.hidden_size, self.num_heads, mlp_ratio=config.mlp_ratio, qkv_bias=config.qkv_bias,
                              fused_qkv=config.fused_qkv) for _ in range(config.depth)])
        self.single_blocks = nn.ModuleList([
            SingleStreamBlock(self.hidden_size, self.num_heads, mlp_ratio=config.mlp_ratio, fused_qkv=config.fused_qkv)
            for _ in range(config.depth_single_blocks)])
        self.final_layer = LastLayer(self.hidden_size, 1, self.out_channels)
        self.initialize_weights()
        self.forward = self.forward_ckpt  # the reference rebinds forward the same way (model.py:143-146)
        self._input_requires_grad = False
        self._cond_w = None
        self._mod_pack = None
        self._mod_lora = None
        self._pe_cache = None
        self._sp_group = None
        self._fp8 = False
        self._fp8_proj = False
        self._fp8_lora = False
        self._fp8_state = None
        self._fp8_attn = False
        self._fp8_attn_state = None
        self.register_load_state_dict_post_hook(lambda m, k: m._drop_caches())

    def _drop_caches(self):
        self._cond_w = self._mod_pack = self._mod_lora = self._pe_cache = None
        self._fp8_state = None   # quantized again from the current parameters at the next forward
        self._fp8_attn_state = None   # workspaces: allocated again on the current device at the next forward

    def _apply(self, fn, *a, **k):
        self._drop_caches()
        return super()._apply(fn, *a, **k)

    # ---- per-step constants (SURVEY.md 8f-2) ------------------------------------------------------------------
    def _grouped_modulation(self, vec: Tensor) -> None:
        """All 2*19 + 38 `Modulation.lin` projections of `vec` as ONE GEMM (the reference launches 76 tiny ones per step,
        layers.py:179-192).  The fp32 result and the column range of every layer ride on `vec`; the processors pick their
        slice (a processor installed on a block this model does not own simply does its own projection).  A layer whose
        active adapters include a DoRA adapter stays out of the group: its magnitude factor scales its base product too,
        which one grouped launch cannot do per layer, so the block projects it itself (osb_gemm_lora with col_scale)."""
        import osb200

        lins = [m.lin for b in self.double_blocks for m in (b.img_mod, b.txt_mod)] + [b.modulation.lin for b in self.single_blocks]
        lins = [lin for lin in lins if all(ad.magnitude is None for ad in adapters_of(lin))]
        if not lins:
            return
        adapted = [lin for lin in lins if adapters_of(lin)]
        key = tuple((id(l), l.weight.data_ptr(), l.weight._version) for l in lins)
        if self._mod_pack is None or self._mod_pack[0] != key:
            cols, off = {}, 0
            for lin in lins:
                cols[id(lin)] = (off, off + lin.out_features)
                off += lin.out_features
            self._mod_pack = (key, torch.cat([l.weight for l in lins], 0).contiguous(),
                              torch.cat([l.bias for l in lins], 0).contiguous(), cols)
        _, w, b, cols = self._mod_pack
        sv = torch.nn.functional.silu(vec).contiguous()
        out = osb200.gemm(sv, w, b)
        if adapted:
            # The base projection keeps its one launch.  Each adapted layer's update is then added into its slice of the
            # bf16 output (R = D, no gate): peft's own two roundings, without a block-diagonal B over every layer and
            # without reading the modulation weights again.  One down projection serves all layers (same input).
            parts = [lora_pack([[(lin, 0, lin.out_features)]]) for lin in adapted]   # per layer (A_cat, [B_cat]), cached
            ml = self._mod_lora
            if ml is None or len(ml[0]) != len(parts) or any(a is not b for a, b in zip(ml[0], parts)):
                self._mod_lora = ml = (parts, torch.cat([p[0] for p in parts], 0).contiguous())
            u = osb200.gemm(sv, ml[1])
            ro = 0
            for lin, (A, (lb,), _) in zip(adapted, parts):
                lo, hi = cols[id(lin)]
                osb200.gemm(u[:, ro:ro + A.shape[0]], lb, None, epilogue=osb200.EPI_BIAS_GATE_RES, residual=out[:, lo:hi],
                            out=out[:, lo:hi])
                ro += A.shape[0]
        vec._osb_grouped_modulation = (out.float(), cols)

    def _pe(self, txt_ids: Tensor, img_ids: Tensor):
        """`pe_embedder(cat(txt_ids, img_ids))` is step-invariant (utils/sampling.py:437-447 builds the ids once per sample):
        cached on the identity and version of the id tensors the caller passes."""
        key = (id(txt_ids), txt_ids._version, id(img_ids), img_ids._version, tuple(txt_ids.shape), tuple(img_ids.shape), txt_ids.device)
        if self._pe_cache is None or self._pe_cache[0] != key:
            # the tensors are kept alive with the entry, so an id() cannot be recycled while it is the key
            self._pe_cache = (key, self.pe_embedder(torch.cat((txt_ids, img_ids), dim=1)), txt_ids, img_ids)
        return self._pe_cache[1]

    def initialize_weights(self):
        if self.config.cond_embed:
            nn.init.zeros_(self.cond_in.weight)
            nn.init.zeros_(self.cond_in.bias)

    def _lin3(self, x: Tensor, lin: nn.Linear, **kw) -> Tensor:
        """Linear over a [B, L, K] tensor; K is zero-padded to a multiple of 8 when needed (cond_in: K = 68)."""
        B, L, K = x.shape
        x2 = x.to(lin.weight.dtype).reshape(B * L, K)
        pad = -K % 8
        w, bias, lora = linear_parts(lin, k_pad=pad)   # the adapter's A is padded along K like the weight
        if pad:
            x2 = torch.nn.functional.pad(x2, (0, pad))
            if self._cond_w is None or self._cond_w[0] is not lin:
                self._cond_w = (lin, torch.nn.functional.pad(lin.weight, (0, pad)).contiguous())
            w = self._cond_w[1]
        import osb200

        x2 = x2.contiguous()
        return _gemm(osb200, x2, w, bias, lora, _down(osb200, x2, lora), **kw).view(B, L, -1)

    def prepare_block_inputs(self, img: Tensor, img_ids: Tensor, txt: Tensor, txt_ids: Tensor, timesteps: Tensor,
                             y_vec: Tensor, cond: Tensor = None, guidance: Tensor | None = None):
        """model.py:154-202."""
        if img.ndim != 3 or txt.ndim != 3:
            raise ValueError("Input img and txt tensors must have 3 dimensions.")
        dt = self.img_in.weight.dtype
        img = self._lin3(img, self.img_in)
        if self.config.cond_embed:
            if cond is None:
                raise ValueError("Didn't get conditional input for conditional model.")
            B, L, C = img.shape
            import osb200

            img = self._lin3(cond, self.cond_in, epilogue=osb200.EPI_BIAS_GATE_RES, residual=img.reshape(B * L, C))
        vec = self.time_in(timestep_embedding(timesteps, 256).to(dt))
        if self.config.guidance_embed:
            if guidance is None:
                raise ValueError("Didn't get guidance strength for guidance distilled model.")
            vec = vec + self.guidance_in(timestep_embedding(guidance, 256).to(dt))
        vec = vec + self.vector_in(y_vec)
        txt = self._lin3(txt, self.txt_in)
        pe = self._pe(txt_ids, img_ids)
        return img, txt, vec, pe

    # ---- FP8 (e4m3) MLPs -------------------------------------------------------------------------------------------
    def _streams(self):
        """(block, kind) of every stream: "img" / "txt" of the double blocks, "single" of the single blocks."""
        return [(b, k) for b in self.double_blocks for k in ("img", "txt")] + [(b, "single") for b in self.single_blocks]

    def _gemm_linears(self, proj: bool) -> list[str]:
        """Names of the Linears that hold the block GEMMs of PROJ_GEMMS (proj) or the other block GEMMs."""
        names = {id(m): n for n, m in self.named_modules()}
        return [names[id(lin)] for blk, kind in self._streams() for gemm, slices in block_gemms(blk, kind).items()
                if (gemm in PROJ_GEMMS) == proj for lin, _, _ in slices]

    def fp8_mlp_linears(self) -> list[str]:
        """Names of the Linears the FP8 path replaces: fc1 / fc2 of the double-block MLPs, and linear1 (or v_mlp) and
        linear2 of the single blocks, which hold their MLP's weights."""
        return self._gemm_linears(False)

    def fp8_proj_linears(self) -> list[str]:
        """Names of the Linears the FP8 projection path (`enable_fp8(projections=True)`) reads: the q|k|v Linears
        (qkv, or q_proj / k_proj / v_proj) and `proj` of both streams of the double blocks, and linear1 (or q_proj /
        k_proj / v_mlp) of the single blocks, which hold their q|k|v rows."""
        return self._gemm_linears(True)

    def enable_fp8(self, projections: bool = False, lora: bool = False) -> None:
        """Run the MLPs of every double and single block on FP8 (e4m3) tensor cores.  The weights are quantized per output
        channel (s = amax / 448) into a per-model cache; the bf16 parameters and the state dict stay as they are.  The fc1
        input is the fp32 LN+modulate row, quantized per row; the fc2 / linear2 input is quantized per 1 x 128 block by
        the fc1 GELU epilogue (and, for the attention half of linear2's input, by osb_quant_blocks_fp8)
        (include/osb200.h, osb_gemm_fp8_blocks).  Needs a hidden size and an MLP width that are multiples of 128 and a
        hidden size of at most 4096 (the FP8 LN+modulate); LoRA / DoRA adapters on the MLP Linears are refused.

        `projections=True` also runs the q|k|v projections and the attention-output `proj` of the double blocks and the
        qkv part of linear1 of the single blocks on FP8: weights per output channel, the q|k|v GEMM input the fp32
        LN+modulate row quantized per row (in a single block the same codes feed its qkv and mlp GEMMs), the `proj` /
        linear2 attention input per 1 x 128 block (by the FP8 attention kernel itself when `enable_fp8_attention()` is on,
        else by osb_quant_blocks_fp8).  Every block Linear then runs on FP8; modulation, embedders and the final layer
        stay bf16.  LoRA / DoRA adapters on those projection Linears (`fp8_proj_linears()`) are refused as well.

        `lora=True` runs LoRA / DoRA adapters on the FP8 Linears instead of refusing them, whether they are loaded
        before or after this call: each adapted GEMM is osb_gemm_fp8_lora, the e4m3 GEMM with the bf16 update
        U (s B)^T (and DoRA's column scale) in the same fp32 accumulator, and U = x A_cat^T is one block-scaled FP8 GEMM per
        shared input that reads the same e4m3 codes as the base GEMM, with lora_A quantized per row (cached per adapter
        state).  This is opt-in because the update then carries FP8 error that the bf16 adapter path does not (e4m3
        activations times an e4m3 copy of lora_A): enabling FP8 never silently changes how a loaded adapter computes.
        With no adapter loaded the output is that of `enable_fp8(projections)`."""
        C, hid = self.hidden_size, int(self.hidden_size * self.config.mlp_ratio)
        if C % 128 or hid % 128:
            raise ValueError(f"FP8 MLPs need the hidden size ({C}) and the MLP width ({hid}) to be multiples of 128 "
                             "(one e4m3 k-block / scale block of osb_gemm_fp8_blocks)")
        if C > 4096:
            raise ValueError(f"FP8 MLPs need a hidden size <= 4096 (the FP8 LN+modulate holds one row), got {C}")
        mods = dict(self.named_modules())
        adapted = [] if lora else [n for n in self.fp8_mlp_linears() if adapters_of(mods[n])]
        if adapted:
            raise ValueError(f"FP8 MLPs cannot run LoRA / DoRA adapters on MLP Linears ({adapted[0]} has one): "
                             "unload_lora first")
        if projections and not lora:
            adapted = [n for n in self.fp8_proj_linears() if adapters_of(mods[n])]
            if adapted:
                raise ValueError(f"FP8 projections cannot run LoRA / DoRA adapters on projection Linears ({adapted[0]} "
                                 "has one): unload_lora first")
        state = Fp8State(projections, lora)
        w = self.img_in.weight
        if w.is_cuda:   # quantized now; a model not yet on the GPU quantizes at its first forward
            import osb200

            for blk, kind in self._streams():
                for name, slices in block_gemms(blk, kind).items():
                    if projections or name not in PROJ_GEMMS:
                        state.weight(osb200, blk, kind, name, slices)
        self._fp8_state, self._fp8, self._fp8_proj, self._fp8_lora = state, True, projections, lora

    def disable_fp8(self) -> None:
        """Back to the bf16 MLPs and projections (adapters on the bf16 LoRA path); the FP8 weight copies and workspaces
        are released."""
        self._fp8, self._fp8_proj, self._fp8_lora, self._fp8_state = False, False, False, None

    # ---- FP8 (e4m3) attention -------------------------------------------------------------------------------------
    def enable_fp8_attention(self) -> None:
        """Run the joint self-attention of every double and single block on FP8 (e4m3) tensor cores (osb_attn_fp8,
        include/osb200.h): q and k quantized per token and head after QK-norm and RoPE, v per channel over the sequence,
        the softmax probabilities as e4m3(256 p).  Independent of `enable_fp8()` (the MLPs): the two compose in either
        order.  No parameter, Linear or adapter changes.  Needs heads of 128 channels."""
        D = self.hidden_size // self.num_heads
        if D != 128:
            raise ValueError(f"FP8 attention needs a head size of 128 (osb_attn_fp8), got {D}")
        self._fp8_attn, self._fp8_attn_state = True, Fp8AttnState()

    def disable_fp8_attention(self) -> None:
        """Back to the bf16 attention (osb_attn_short); the FP8 attention workspaces are released."""
        self._fp8_attn, self._fp8_attn_state = False, None

    def enable_sequence_parallel(self, group) -> None:
        """Ulysses sequence parallelism over `group` (the reference's `all_to_all` mode, opensora/models/mmdit/
        distributed.py:473-495,598-634,671-679): the joint txt|img sequence is split into P equal chunks (a rank holds the tail
        of the text and/or a slice of the image tokens), every token-local op runs on the chunk, attention exchanges
        "scatter heads / gather sequence" on q|k|v (ONE all-to-all for the three) and back on the output, and the image
        tokens are all-gathered (var-len) after the final layer.  `None` switches it off."""
        self._sp_group = group

    def _sp_splits(self, Lt: int, Li: int):
        """(P, rank, [txt tokens per rank], [img tokens per rank]) of the equal split of the joint sequence, or None when
        sequence parallelism is off / not applicable (distributed.py:604-617: a rank without image tokens disables it)."""
        import torch.distributed as dist

        g = getattr(self, "_sp_group", None)
        if g is None or not dist.is_initialized() or dist.get_world_size(g) == 1:
            return None
        P, r = dist.get_world_size(g), dist.get_rank(g)
        if (Lt + Li) % P:
            raise ValueError(f"Expected {Lt + Li} % {P} == 0 (distributed.py:600-604)")
        ch = (Lt + Li) // P
        txt_s = [max(0, min((k + 1) * ch, Lt) - min(k * ch, Lt)) for k in range(P)]
        img_s = [ch - t for t in txt_s]
        if 0 in img_s:
            return None
        return P, r, txt_s, img_s

    def forward_ckpt(self, img: Tensor, img_ids: Tensor, txt: Tensor, txt_ids: Tensor, timesteps: Tensor, y_vec: Tensor,
                     cond: Tensor = None, guidance: Tensor | None = None, **kwargs) -> Tensor:
        """model.py:208-233; with a sequence-parallel group: distributed.py:598-681 (forward part)."""
        from . import layers as L_

        img, txt, vec, pe = self.prepare_block_inputs(img, img_ids, txt, txt_ids, timesteps, y_vec, cond, guidance)
        self._grouped_modulation(vec)
        if self._fp8:
            if self._fp8_state is None:
                self._fp8_state = Fp8State(self._fp8_proj, self._fp8_lora)
            vec._osb_fp8 = self._fp8_state
        if self._fp8_attn:
            if self._fp8_attn_state is None:
                self._fp8_attn_state = Fp8AttnState()
            vec._osb_fp8_attn = self._fp8_attn_state
        Lt, Li = txt.shape[1], img.shape[1]
        sp = self._sp_splits(Lt, Li)
        vec._osb_txt_len = Lt   # joint positions >= Lt take the image stream's QK-norm weights on every rank
        if sp is not None:
            P, r, txt_s, img_s = sp
            t0, i0 = sum(txt_s[:r]), sum(img_s[:r])
            txt, img = txt[:, t0:t0 + txt_s[r]].contiguous(), img[:, i0:i0 + img_s[r]].contiguous()
        prev = L_._SP["group"]
        L_._SP["group"] = self._sp_group if sp is not None else None
        try:
            for block in self.double_blocks:
                img, txt = block(img, txt, vec, pe)
            x = torch.cat((txt, img), 1)
            for block in self.single_blocks:
                x = block(x, vec, pe)
        finally:
            L_._SP["group"] = prev
        out = self.final_layer(x[:, txt.shape[1]:, ...].contiguous(), vec)
        if sp is not None:
            from opensora.acceleration.communications import gather_forward_split_backward_var_len

            out = gather_forward_split_backward_var_len(out, 1, self._sp_group, sp[3])
        return out

    forward_selective_ckpt = forward_ckpt


@MODELS.register_module("flux")
def Flux(cache_dir: str = None, from_pretrained: str = None, device_map: str | torch.device = "cuda",
         torch_dtype: torch.dtype = torch.bfloat16, strict_load: bool = False, **kwargs) -> MMDiTModel:
    """model.py:271-303.  Weights go through `opensora.utils.ckpt.load_checkpoint` like upstream (safetensors / torch file /
    sharded directory; local or hub-cache paths only - no network here)."""
    config = MMDiTConfig(from_pretrained=from_pretrained, cache_dir=cache_dir, **kwargs)
    model = MMDiTModel(config)
    if from_pretrained:
        from opensora.utils.ckpt import load_checkpoint

        model = load_checkpoint(model, from_pretrained, cache_dir=cache_dir, device_map="cpu", strict=strict_load)
    return model.to(device=device_map, dtype=torch_dtype)
