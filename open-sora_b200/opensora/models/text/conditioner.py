"""Drop-in for the reference's `opensora/models/text/conditioner.py:10-53`: `HFEmbedder`, registered as "text_embedder",
turns prompts into the denoiser's text inputs.  T5 v1.1 (gated GELU) gives `last_hidden_state` [B, L, d_model]
(`txt`), CLIP's text transformer gives `pooler_output` [B, hidden] (`y_vec`).

The encoders run on osb200 kernels; the model code needs no transformers.  Weights come from the checkpoint
directory through `opensora.utils.ckpt.load_checkpoint` (safetensors, sharded index or .bin) under their Hugging Face
key names, and `config.json` is read as JSON.  Only tokenization imports transformers, lazily and offline.

  T5 layer:   RMSNorm -> one q|k|v GEMM -> attention with the relative-position bias of block 0 (unscaled scores) ->
              o-projection + residual -> RMSNorm -> gated-GELU GEMM over interleaved wi_0 / wi_1 -> wo + residual;
              final RMSNorm.
  CLIP layer: LayerNorm (osb_ln_modulate with scale = w - 1, shift = b) -> q|k|v GEMM + bias -> causal attention (a
              0 / -inf bias vector) -> out_proj + residual -> LayerNorm -> fc1 + quick GELU -> fc2 + residual; final
              LayerNorm of the pooled row only (LayerNorm is per row).

The token-embedding gather and CLIP's position-embedding add are torch ops.  The forward after tokenization
(`encode`) is CUDA-graph capturable once the bias vector of its length is cached (the first eager call caches it).
`shardformer=True` is accepted for T5 and changes no arithmetic: the ColossalAI policy of the reference only jit-fuses
the dropout-add and the feed-forward forward (opensora/acceleration/shardformer/policy/t5_encoder.py)."""
from __future__ import annotations

import json
import math
import os

import torch
import torch.nn as nn
import torch.nn.functional as F

from opensora.registry import MODELS
from opensora.utils.ckpt import load_checkpoint

HEAD_DIM = 64   # the only head size the bias attention kernel is built for

# transformers' T5Config / CLIPTextConfig defaults for keys a config.json may leave out
_T5_DEFAULTS = dict(vocab_size=32128, d_model=512, d_kv=64, d_ff=2048, num_layers=6, num_heads=8,
                    relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
                    feed_forward_proj="relu")
_CLIP_DEFAULTS = dict(vocab_size=49408, hidden_size=512, intermediate_size=2048, num_hidden_layers=12,
                      num_attention_heads=8, max_position_embeddings=77, hidden_act="quick_gelu", layer_norm_eps=1e-5,
                      eos_token_id=2)


def _osb():
    import osb200

    return osb200


def relative_position_bucket(relative_position: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """T5's bidirectional `_relative_position_bucket` (transformers T5Attention), with the same float ops, so no bucket
    boundary moves.  relative_position = key position - query position (int64)."""
    num_buckets //= 2
    buckets = (relative_position > 0).to(torch.long) * num_buckets
    relative_position = torch.abs(relative_position)
    max_exact = num_buckets // 2
    is_small = relative_position < max_exact
    large = max_exact + (
        torch.log(relative_position.float() / max_exact) / math.log(max_distance / max_exact) * (num_buckets - max_exact)
    ).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return buckets + torch.where(is_small, relative_position, large)


def clip_ln_scale(w: torch.Tensor, name: str) -> torch.Tensor:
    """LayerNorm weight -> the `scale` of osb_ln_modulate, which multiplies by 1 + scale in fp32.  1 + (w - 1) == w in
    fp32 for every bf16 w with w == 0 or 2^-16 <= |w| < 2^16, so the affine LayerNorm is computed exactly; a weight
    outside that range is refused, naming the layer."""
    wf = w.float()
    a = wf.abs()
    bad = ~((wf == 0) | ((a >= 2.0 ** -16) & (a < 2.0 ** 16)))
    if bool(bad.any()):
        raise _osb().OsbError(f"{name}: LayerNorm weight {float(wf[bad][0])} is outside 0 or [2^-16, 2^16) in magnitude; "
                              "osb_ln_modulate cannot apply it exactly")
    return (wf - 1.0).reshape(1, -1).contiguous()


class _Checkpoint(nn.Module):
    """The checkpoint's tensors under their HF key names, with the expected shapes.  `load_state_dict` drops the keys
    the encoder never reads (`ignore(key)`) and is strict about the rest: a missing, unexpected or mis-shaped key
    raises, naming the key.  Parameters start on the meta device and are replaced by the loaded tensors."""

    def __init__(self, shapes: dict[str, tuple], ignore):
        super().__init__()
        self._ignore = ignore
        for key, shape in shapes.items():
            *path, leaf = key.split(".")
            mod = self
            for p in path:
                if not hasattr(mod, p):
                    mod.add_module(p, nn.Module())
                mod = getattr(mod, p)
            mod.register_parameter(leaf, nn.Parameter(torch.empty(shape, device="meta"), requires_grad=False))

    def load_state_dict(self, state_dict, strict: bool = True, assign: bool = False):
        sd = {k: v for k, v in state_dict.items() if not self._ignore(k)}
        return super().load_state_dict(sd, strict=True, assign=True)


def _t5_shapes(c: dict) -> dict[str, tuple]:
    d, inner, ff, H = c["d_model"], c["num_heads"] * c["d_kv"], c["d_ff"], c["num_heads"]
    s = {"shared.weight": (c["vocab_size"], d), "encoder.final_layer_norm.weight": (d,),
         "encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight": (c["relative_attention_num_buckets"], H)}
    for i in range(c["num_layers"]):
        b = f"encoder.block.{i}.layer."
        for n in "qkv":
            s[f"{b}0.SelfAttention.{n}.weight"] = (inner, d)
        s[f"{b}0.SelfAttention.o.weight"] = (d, inner)
        s[f"{b}0.layer_norm.weight"] = (d,)
        s[f"{b}1.DenseReluDense.wi_0.weight"] = (ff, d)
        s[f"{b}1.DenseReluDense.wi_1.weight"] = (ff, d)
        s[f"{b}1.DenseReluDense.wo.weight"] = (d, ff)
        s[f"{b}1.layer_norm.weight"] = (d,)
    return s


def _t5_ignored(key: str) -> bool:
    # a T5ForConditionalGeneration checkpoint also holds the decoder and LM head; embed_tokens is tied to `shared`
    return key.startswith(("decoder.", "lm_head.")) or key == "encoder.embed_tokens.weight"


def _clip_shapes(c: dict) -> dict[str, tuple]:
    d, ff = c["hidden_size"], c["intermediate_size"]
    p = "text_model."
    s = {f"{p}embeddings.token_embedding.weight": (c["vocab_size"], d),
         f"{p}embeddings.position_embedding.weight": (c["max_position_embeddings"], d),
         f"{p}final_layer_norm.weight": (d,), f"{p}final_layer_norm.bias": (d,)}
    for i in range(c["num_hidden_layers"]):
        b = f"{p}encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            s[f"{b}self_attn.{n}.weight"] = (d, d)
            s[f"{b}self_attn.{n}.bias"] = (d,)
        for n in ("layer_norm1", "layer_norm2"):
            s[f"{b}{n}.weight"] = (d,)
            s[f"{b}{n}.bias"] = (d,)
        s[f"{b}mlp.fc1.weight"] = (ff, d)
        s[f"{b}mlp.fc1.bias"] = (ff,)
        s[f"{b}mlp.fc2.weight"] = (d, ff)
        s[f"{b}mlp.fc2.bias"] = (d,)
    return s


def _clip_ignored(key: str) -> bool:
    # a CLIPModel checkpoint also holds the vision tower and the projections
    return not key.startswith("text_model.") or key == "text_model.embeddings.position_ids"


def read_config(path: str, is_clip: bool) -> dict:
    """config.json of the checkpoint directory with transformers' defaults filled in; unsupported models are refused."""
    with open(os.path.join(path, "config.json")) as fh:
        raw = json.load(fh)
    err = _osb().OsbError
    if is_clip:
        c = dict(_CLIP_DEFAULTS, **raw.get("text_config", raw))
        if c["hidden_act"] != "quick_gelu":
            raise err(f"{path}: CLIP hidden_act {c['hidden_act']!r} is not supported (quick_gelu only)")
        if c["hidden_size"] != c["num_attention_heads"] * HEAD_DIM:
            raise err(f"{path}: CLIP head size {c['hidden_size'] / c['num_attention_heads']:g} is not supported "
                      f"({HEAD_DIM} only)")
        if c["hidden_size"] % 8 or c["intermediate_size"] % 8:
            raise err(f"{path}: CLIP widths must be multiples of 8")
    else:
        c = dict(_T5_DEFAULTS, **raw)
        if c["feed_forward_proj"] != "gated-gelu":
            raise err(f"{path}: T5 feed_forward_proj {c['feed_forward_proj']!r} is not supported: only the gated-GELU "
                      "T5 v1.1 encoder is (T5 v1.0 uses relu)")
        if c["d_kv"] != HEAD_DIM:
            raise err(f"{path}: T5 head size d_kv = {c['d_kv']} is not supported ({HEAD_DIM} only)")
        if c["d_model"] % 8 or c["d_ff"] % 8:
            raise err(f"{path}: T5 widths must be multiples of 8")
    return c


def _layer(**tensors) -> nn.Module:
    m = nn.Module()
    for k, v in tensors.items():
        m.register_buffer(k, v, persistent=False)
    return m


@MODELS.register_module("text_embedder")
class HFEmbedder(nn.Module):
    """`HFEmbedder(from_pretrained, max_length, shardformer=False, device_map=..., torch_dtype=...)`: a CLIP text encoder
    when the path names "openai" (as the reference decides), else a T5 v1.1 encoder.  bf16 only; the forward runs on
    CUDA only.  `tokenizer=` replaces the tokenizer loaded from the checkpoint directory."""

    def __init__(self, from_pretrained: str, max_length: int, shardformer: bool = False, device_map=None,
                 torch_dtype: torch.dtype | None = None, tokenizer=None):
        super().__init__()
        osb = _osb()
        self.is_clip = "openai" in from_pretrained
        self.max_length = max_length
        self.output_key = "pooler_output" if self.is_clip else "last_hidden_state"
        self.from_pretrained = from_pretrained
        if torch_dtype is not None and torch_dtype != torch.bfloat16:
            raise osb.OsbError(f"text_embedder runs in bfloat16 only, got torch_dtype={torch_dtype}")
        if self.is_clip:
            assert not shardformer, "Shardformer is not supported for CLIP"
        self._tokenizer = tokenizer
        device = torch.device(device_map) if device_map is not None else torch.device("cpu")
        cfg = read_config(from_pretrained, self.is_clip)
        self.config = cfg
        ck = _Checkpoint(_clip_shapes(cfg) if self.is_clip else _t5_shapes(cfg),
                         _clip_ignored if self.is_clip else _t5_ignored)
        load_checkpoint(ck, from_pretrained, strict=True)
        w = {k: v.detach() for k, v in ck.named_parameters()}
        del ck

        def bf(key):
            return w.pop(key).to(device=device, dtype=torch.bfloat16).contiguous()

        self.layers = nn.ModuleList()
        if self.is_clip:
            p = "text_model."
            self.num_heads = cfg["num_attention_heads"]
            self.eps = cfg["layer_norm_eps"]
            self.eos_token_id = cfg["eos_token_id"]
            self.register_buffer("tok_emb", bf(f"{p}embeddings.token_embedding.weight"), persistent=False)
            self.register_buffer("pos_emb", bf(f"{p}embeddings.position_embedding.weight"), persistent=False)

            def ln(name):
                scale = clip_ln_scale(bf(f"{name}.weight"), name).to(device)
                return scale, bf(f"{name}.bias").float().reshape(1, -1).contiguous()

            for i in range(cfg["num_hidden_layers"]):
                b = f"{p}encoder.layers.{i}."
                s1, h1 = ln(f"{b}layer_norm1")
                s2, h2 = ln(f"{b}layer_norm2")
                qkv_w = torch.cat([bf(f"{b}self_attn.{n}_proj.weight") for n in "qkv"]).contiguous()
                qkv_b = torch.cat([bf(f"{b}self_attn.{n}_proj.bias") for n in "qkv"]).contiguous()
                self.layers.append(_layer(ln1_scale=s1, ln1_shift=h1, qkv_w=qkv_w, qkv_b=qkv_b,
                                          o_w=bf(f"{b}self_attn.out_proj.weight"), o_b=bf(f"{b}self_attn.out_proj.bias"),
                                          ln2_scale=s2, ln2_shift=h2, fc1_w=bf(f"{b}mlp.fc1.weight"),
                                          fc1_b=bf(f"{b}mlp.fc1.bias"), fc2_w=bf(f"{b}mlp.fc2.weight"),
                                          fc2_b=bf(f"{b}mlp.fc2.bias")))
            fs, fh = ln(f"{p}final_layer_norm")
            self.register_buffer("final_scale", fs, persistent=False)
            self.register_buffer("final_shift", fh, persistent=False)
        else:
            self.num_heads = cfg["num_heads"]
            self.eps = cfg["layer_norm_epsilon"]
            self.num_buckets = cfg["relative_attention_num_buckets"]
            self.max_distance = cfg["relative_attention_max_distance"]
            self.register_buffer("shared", bf("shared.weight"), persistent=False)
            # block 0's table serves every layer; kept on the host, where the per-length bias vectors are gathered
            self.rel_table = w.pop("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight").to(torch.bfloat16).float()
            for i in range(cfg["num_layers"]):
                b = f"encoder.block.{i}.layer."
                qkv_w = torch.cat([bf(f"{b}0.SelfAttention.{n}.weight") for n in "qkv"]).contiguous()
                wi = osb.interleave_gated(bf(f"{b}1.DenseReluDense.wi_0.weight"), bf(f"{b}1.DenseReluDense.wi_1.weight"))
                self.layers.append(_layer(ln0=bf(f"{b}0.layer_norm.weight"), qkv_w=qkv_w, o_w=bf(f"{b}0.SelfAttention.o.weight"),
                                          ln1=bf(f"{b}1.layer_norm.weight"), wi=wi, wo=bf(f"{b}1.DenseReluDense.wo.weight")))
            self.register_buffer("final_ln", bf("encoder.final_layer_norm.weight"), persistent=False)
        assert not w, f"unused checkpoint tensors: {sorted(w)}"
        self._bias: dict[int, torch.Tensor] = {}
        self.eval().requires_grad_(False)

    # ---- tokenization (host plumbing) --------------------------------------------------------------------------------
    @property
    def tokenizer(self):
        if self._tokenizer is None:
            if self.is_clip:
                from transformers import CLIPTokenizer

                self._tokenizer = CLIPTokenizer.from_pretrained(self.from_pretrained, max_length=self.max_length,
                                                                local_files_only=True)
            else:
                from transformers import T5Tokenizer

                self._tokenizer = T5Tokenizer.from_pretrained(self.from_pretrained, max_length=self.max_length,
                                                              legacy=True, local_files_only=True)
        return self._tokenizer

    def tokenize(self, text: list[str], added_tokens: int = 0, seq_align: int = 1) -> torch.Tensor:
        """Token ids [B, L] as the reference builds them: padded to max_length with truncation, then right-padded with
        pad_token_id until added_tokens + L is a multiple of seq_align."""
        enc = self.tokenizer(text, truncation=True, max_length=self.max_length, return_length=False,
                             return_overflowing_tokens=False, padding="max_length", return_tensors="pt")
        ids = enc["input_ids"]
        seq_len = ids.shape[1]
        if (added_tokens + seq_len) % seq_align != 0:
            num_pad = seq_align - (added_tokens + seq_len) % seq_align
            ids = F.pad(ids, (0, num_pad), value=self.tokenizer.pad_token_id)
        return ids

    def forward(self, text: list[str], added_tokens: int = 0, seq_align: int = 1) -> torch.Tensor:
        ids = self.tokenize(text, added_tokens, seq_align)
        return self.encode(ids.to(self._weight().device))

    # ---- encoders ----------------------------------------------------------------------------------------------------
    def _weight(self) -> torch.Tensor:
        return self.tok_emb if self.is_clip else self.shared

    def attn_bias(self, L: int) -> torch.Tensor:
        """Cached fp32 bias vector of osb_attn_short_bias for L tokens: T5 [H, 2L - 1] = table[bucket(j - i)], CLIP
        [2L - 1] = 0 for j <= i, -inf for j > i (index j - i + L - 1)."""
        b = self._bias.get(L)
        if b is None:
            rel = torch.arange(-(L - 1), L, dtype=torch.long)
            if self.is_clip:
                b = torch.where(rel > 0, float("-inf"), 0.0).float()
            else:
                b = self.rel_table[relative_position_bucket(rel, self.num_buckets, self.max_distance)].t().contiguous()
            b = b.to(self._weight().device)
            self._bias[L] = b
        return b

    def encode(self, ids: torch.Tensor) -> torch.Tensor:
        """Token ids [B, L] on the model's device -> T5 last_hidden_state [B, L, d_model] or CLIP pooler_output [B, d]."""
        osb = _osb()
        osb.require_cuda_bf16(self._weight(), "text_embedder")
        if ids.device != self._weight().device:
            raise osb.OsbError(f"text_embedder: input_ids on {ids.device}, model on {self._weight().device}")
        return self._clip(ids) if self.is_clip else self._t5(ids)

    def _attention(self, qkv: torch.Tensor, B: int, L: int, scale: float) -> torch.Tensor:
        osb = _osb()
        inner = self.num_heads * HEAD_DIM
        out = torch.empty(B * L, inner, dtype=qkv.dtype, device=qkv.device)
        return osb.attn_short_bias(qkv[:, :inner], qkv[:, inner:2 * inner], qkv[:, 2 * inner:], out, self.attn_bias(L),
                                   num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L,
                                   num_heads=self.num_heads, head_dim=HEAD_DIM, softmax_scale=scale)

    def _t5(self, ids: torch.Tensor) -> torch.Tensor:
        osb = _osb()
        B, L = ids.shape
        x = F.embedding(ids, self.shared).reshape(B * L, -1).contiguous()
        for lay in self.layers:
            h = osb.rms_norm(x, lay.ln0, eps=self.eps)
            a = self._attention(osb.gemm(h, lay.qkv_w), B, L, 1.0)   # T5 does not scale its scores
            x = osb.gemm(a, lay.o_w, epilogue=osb.EPI_BIAS_GATE_RES, residual=x, out=x)
            h = osb.rms_norm(x, lay.ln1, eps=self.eps)
            f = osb.gemm(h, lay.wi, epilogue=osb.EPI_GATED_GELU)
            x = osb.gemm(f, lay.wo, epilogue=osb.EPI_BIAS_GATE_RES, residual=x, out=x)
        return osb.rms_norm(x, self.final_ln, eps=self.eps).view(B, L, -1)

    def _clip(self, ids: torch.Tensor) -> torch.Tensor:
        osb = _osb()
        B, L = ids.shape
        x = (F.embedding(ids, self.tok_emb) + self.pos_emb[:L]).reshape(B * L, -1).contiguous()
        M = B * L
        for lay in self.layers:
            h = osb.ln_modulate(x, lay.ln1_shift, lay.ln1_scale, group_rows=M, eps=self.eps)
            a = self._attention(osb.gemm(h, lay.qkv_w, lay.qkv_b), B, L, HEAD_DIM ** -0.5)
            x = osb.gemm(a, lay.o_w, lay.o_b, epilogue=osb.EPI_BIAS_GATE_RES, residual=x, out=x)
            h = osb.ln_modulate(x, lay.ln2_shift, lay.ln2_scale, group_rows=M, eps=self.eps)
            f = osb.gemm(h, lay.fc1_w, lay.fc1_b, epilogue=osb.EPI_BIAS_QUICK_GELU)
            x = osb.gemm(f, lay.fc2_w, lay.fc2_b, epilogue=osb.EPI_BIAS_GATE_RES, residual=x, out=x)
        ids32 = ids.to(torch.int)
        if self.eos_token_id == 2:   # legacy configs (openai/clip-vit-large-patch14): the eos token has the largest id
            eos = ids32.argmax(dim=-1)
        else:
            eos = (ids32 == self.eos_token_id).int().argmax(dim=-1)
        pooled = x.view(B, L, -1)[torch.arange(B, device=x.device), eos].contiguous()
        return osb.ln_modulate(pooled, self.final_shift, self.final_scale, group_rows=B, eps=self.eps)
