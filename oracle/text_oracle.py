"""ORACLE - functional restatement of the reference's text encoders as `text_embedder` runs them (HF T5EncoderModel of
T5 v1.1 and CLIPTextModel, opensora/models/text/conditioner.py:10-53, attention_mask=None).  Weights are a dict under
the Hugging Face key names.  In fp32 this is the parity reference; with dtype=torch.bfloat16 every op rounds where the
reference's bf16 modules round (matmul outputs, residual adds, T5LayerNorm's two roundings, softmax in fp32 cast back),
which gives the bf16 noise floor and the eager-torch baseline of the benchmark."""
from __future__ import annotations

import math

import torch
import torch.nn.functional as F


def t5_bucket(rel: torch.Tensor, num_buckets: int = 32, max_distance: int = 128) -> torch.Tensor:
    """Bidirectional relative-position bucket of T5Attention._relative_position_bucket."""
    num_buckets //= 2
    out = (rel > 0).to(torch.long) * num_buckets
    n = torch.abs(rel)
    max_exact = num_buckets // 2
    large = max_exact + (torch.log(n.float() / max_exact) / math.log(max_distance / max_exact)
                         * (num_buckets - max_exact)).to(torch.long)
    large = torch.min(large, torch.full_like(large, num_buckets - 1))
    return out + torch.where(n < max_exact, n, large)


def _rms(x, w, eps, dtype):
    var = x.float().pow(2).mean(-1, keepdim=True)
    return w * (x * torch.rsqrt(var + eps)).to(dtype)


def t5_encode(w: dict, cfg: dict, ids: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """last_hidden_state [B, L, d_model] of the T5 v1.1 encoder."""
    dev = ids.device
    g = lambda k: w[k].to(dev, dtype)   # noqa: E731
    B, L = ids.shape
    H, dk, eps = cfg["num_heads"], cfg["d_kv"], cfg.get("layer_norm_epsilon", 1e-6)
    x = F.embedding(ids, g("shared.weight"))
    pos = torch.arange(L, device=dev)
    bucket = t5_bucket(pos[None, :] - pos[:, None], cfg.get("relative_attention_num_buckets", 32),
                       cfg.get("relative_attention_max_distance", 128))
    bias = g("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")[bucket].permute(2, 0, 1)[None]
    for i in range(cfg["num_layers"]):
        p = f"encoder.block.{i}.layer."
        h = _rms(x, g(p + "0.layer_norm.weight"), eps, dtype)
        q, k, v = (F.linear(h, g(f"{p}0.SelfAttention.{n}.weight")).view(B, L, H, dk).transpose(1, 2) for n in "qkv")
        s = q @ k.transpose(-1, -2) + bias
        a = torch.softmax(s.float(), dim=-1).to(dtype)
        o = (a @ v).transpose(1, 2).reshape(B, L, H * dk)
        x = x + F.linear(o, g(p + "0.SelfAttention.o.weight"))
        h = _rms(x, g(p + "1.layer_norm.weight"), eps, dtype)
        f = F.gelu(F.linear(h, g(p + "1.DenseReluDense.wi_0.weight")), approximate="tanh") * F.linear(
            h, g(p + "1.DenseReluDense.wi_1.weight"))
        x = x + F.linear(f, g(p + "1.DenseReluDense.wo.weight"))
    return _rms(x, g("encoder.final_layer_norm.weight"), eps, dtype)


def clip_pool_index(ids: torch.Tensor, eos_token_id: int) -> torch.Tensor:
    """CLIPTextTransformer's pooled position: argmax(ids) for legacy configs (eos_token_id == 2), else the first eos."""
    ids = ids.to(torch.int)
    if eos_token_id == 2:
        return ids.argmax(dim=-1)
    return (ids == eos_token_id).int().argmax(dim=-1)


def clip_encode(w: dict, cfg: dict, ids: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """pooler_output [B, hidden] of the CLIP text transformer (quick_gelu, causal self-attention)."""
    dev = ids.device
    g = lambda k: w["text_model." + k].to(dev, dtype)   # noqa: E731
    B, L = ids.shape
    H = cfg["num_attention_heads"]
    d = cfg["hidden_size"]
    dk, eps = d // H, cfg.get("layer_norm_eps", 1e-5)
    x = F.embedding(ids, g("embeddings.token_embedding.weight")) + g("embeddings.position_embedding.weight")[:L]
    mask = torch.full((L, L), float("-inf"), device=dev).triu(1).to(dtype)
    for i in range(cfg["num_hidden_layers"]):
        p = f"encoder.layers.{i}."
        h = F.layer_norm(x, (d,), g(p + "layer_norm1.weight"), g(p + "layer_norm1.bias"), eps)
        q, k, v = (F.linear(h, g(f"{p}self_attn.{n}_proj.weight"), g(f"{p}self_attn.{n}_proj.bias"))
                   .view(B, L, H, dk).transpose(1, 2) for n in "qkv")
        s = (q @ k.transpose(-1, -2)) * dk ** -0.5 + mask
        a = torch.softmax(s.float(), dim=-1).to(dtype)
        o = (a @ v).transpose(1, 2).reshape(B, L, d)
        x = x + F.linear(o, g(p + "self_attn.out_proj.weight"), g(p + "self_attn.out_proj.bias"))
        h = F.layer_norm(x, (d,), g(p + "layer_norm2.weight"), g(p + "layer_norm2.bias"), eps)
        f = F.linear(h, g(p + "mlp.fc1.weight"), g(p + "mlp.fc1.bias"))
        f = f * torch.sigmoid(1.702 * f)
        x = x + F.linear(f, g(p + "mlp.fc2.weight"), g(p + "mlp.fc2.bias"))
    x = F.layer_norm(x, (d,), g("final_layer_norm.weight"), g("final_layer_norm.bias"), eps)
    return x[torch.arange(B, device=dev), clip_pool_index(ids, cfg.get("eos_token_id", 2))]
