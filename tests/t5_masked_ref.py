"""fp32 / bf16 restatement of transformers' T5EncoderModel(input_ids, attention_mask) for the v1.2 T5 tests: the T5 v1.1
encoder of `oracle.text_oracle.t5_encode` (same bucket function, T5LayerNorm roundings and rounding points) with the
attention mask applied as transformers applies it - the dtype's lowest value added to the bias of every masked key in
every layer, every query row still computed.  With an all-ones mask it computes exactly what `t5_encode` computes
(tests/test_t5_v12_cpu.py); with a mask it is pinned to tests/golden/t5_masked.npz."""
from __future__ import annotations

import torch
import torch.nn.functional as F

from oracle.text_oracle import _rms, t5_bucket


def t5_encode_masked(w: dict, cfg: dict, ids: torch.Tensor, mask: torch.Tensor, dtype=torch.float32) -> torch.Tensor:
    """last_hidden_state [B, L, d_model]; `mask` [B, L], 1 = token, 0 = pad."""
    dev = ids.device
    g = lambda k: w[k].to(dev, dtype)   # noqa: E731
    B, L = ids.shape
    H, dk, eps = cfg["num_heads"], cfg["d_kv"], cfg.get("layer_norm_epsilon", 1e-6)
    x = F.embedding(ids, g("shared.weight"))
    pos = torch.arange(L, device=dev)
    bucket = t5_bucket(pos[None, :] - pos[:, None], cfg.get("relative_attention_num_buckets", 32),
                       cfg.get("relative_attention_max_distance", 128))
    bias = g("encoder.block.0.layer.0.SelfAttention.relative_attention_bias.weight")[bucket].permute(2, 0, 1)[None]
    bias = bias + (1.0 - mask.to(dev, dtype))[:, None, None, :] * torch.finfo(dtype).min
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
