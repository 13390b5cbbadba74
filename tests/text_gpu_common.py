"""Random-weight text encoders on the GPU for the text_embedder GPU tests and benchmark: weights generated on the device
(transformers' _init_weights scales for the full-size models) and handed to `HFEmbedder` through its checkpoint loader,
so the model is built by the same code path as from a checkpoint directory, without writing gigabytes to disk."""
from __future__ import annotations

import json
import os

import torch


def device_weights(shapes: dict, is_clip: bool, seed: int, d_model: int) -> dict[str, torch.Tensor]:
    """bf16 weights on cuda.  CLIP: transformers' CLIPPreTrainedModel._init_weights with initializer_factor 1 (token /
    position embeddings N(0, 0.02), q/k/v/out N(0, d^-0.5 L2^-1/2 ...)), LayerNorm weight 1 and bias 0 perturbed by
    N(0, 0.05) so the affine path is exercised.  T5: T5PreTrainedModel._init_weights (shared N(0, 1), q N(0, (d d_kv)^-1/2),
    k / v / o / wi / wo N(0, fan_in^-1/2), relative bias N(0, d^-1/2)), norms 1 + N(0, 0.05)."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = {}
    for key in sorted(shapes):
        shape = shapes[key]
        r = torch.randn(shape, generator=g, device="cuda")
        if "norm" in key and key.endswith("weight"):
            t = 1.0 + 0.05 * r
        elif "norm" in key:
            t = 0.05 * r
        elif key.endswith("bias") and "relative" not in key:
            t = torch.zeros_like(r)
        elif "relative_attention_bias" in key:
            t = r * d_model ** -0.5
        elif "embedding" in key:
            t = 0.02 * r
        elif key == "shared.weight":
            t = r
        elif is_clip and "fc" in key:
            t = r * (shape[1] ** -0.5)
        elif is_clip:
            t = r * d_model ** -0.5
        elif key.endswith("q.weight"):
            t = r * (d_model * 64) ** -0.25 * d_model ** -0.25
        else:
            t = r * shape[1] ** -0.5
        out[key] = t.to(torch.bfloat16)
        del r
    return out


def build(tmp_dir: str, cfg: dict, weights: dict, is_clip: bool, max_length: int, tokenizer=None):
    """HFEmbedder on cuda from in-memory weights: config.json is written to `tmp_dir`, the checkpoint loader is given
    the tensors instead of reading files."""
    from opensora.models.text import conditioner

    d = os.path.join(tmp_dir, "openai" if is_clip else "google", "model")
    os.makedirs(d, exist_ok=True)
    with open(os.path.join(d, "config.json"), "w") as fh:
        json.dump(cfg, fh)
    real = conditioner.load_checkpoint
    conditioner.load_checkpoint = lambda model, path, **kw: model.load_state_dict(weights, strict=True)
    try:
        return conditioner.HFEmbedder(d, max_length=max_length, device_map="cuda", torch_dtype=torch.bfloat16,
                                      tokenizer=tokenizer)
    finally:
        conditioner.load_checkpoint = real


def encoder_parity(name, out, fp32, bf16, cap):
    err = float((out.float() - fp32).norm() / fp32.norm())
    floor = float((bf16.float() - fp32).norm() / fp32.norm())
    print(f"{name}: rel-L2 error {err:.3e}, bf16 floor {floor:.3e}, ratio {err / floor:.3f}")
    assert err <= 1.1 * floor and err < cap, (name, err, floor)
