"""Seeded toy text encoders for the text_embedder tests and goldens: configs, weights under Hugging Face key names
(generated from a seed with torch, so the goldens store only seeds, configs, token ids and outputs), a checkpoint
directory writer and a deterministic toy tokenizer (prompts are space-separated token ids)."""
from __future__ import annotations

import json
import os

import torch

T5_TINY = dict(model_type="t5", vocab_size=384, d_model=128, d_kv=64, d_ff=320, num_layers=2, num_heads=2,
               relative_attention_num_buckets=32, relative_attention_max_distance=128, layer_norm_epsilon=1e-6,
               feed_forward_proj="gated-gelu", is_encoder_decoder=False, use_cache=False, tie_word_embeddings=False)
CLIP_TINY = dict(model_type="clip_text_model", vocab_size=320, hidden_size=128, intermediate_size=256,
                 num_hidden_layers=2, num_attention_heads=2, max_position_embeddings=77, hidden_act="quick_gelu",
                 layer_norm_eps=1e-5, bos_token_id=318, eos_token_id=2, pad_token_id=1)
T5_XXL = dict(T5_TINY, vocab_size=32128, d_model=4096, d_ff=10240, num_layers=24, num_heads=64)
CLIP_L = dict(CLIP_TINY, vocab_size=49408, hidden_size=768, intermediate_size=3072, num_hidden_layers=12,
              num_attention_heads=12, bos_token_id=49406)
SEED_T5, SEED_CLIP = 1234, 4321


def t5_weights(cfg: dict, seed: int) -> dict[str, torch.Tensor]:
    from opensora.models.text.conditioner import _t5_shapes

    return _seeded(_t5_shapes(dict(cfg)), seed, is_clip=False)


def clip_weights(cfg: dict, seed: int) -> dict[str, torch.Tensor]:
    from opensora.models.text.conditioner import _clip_shapes

    return _seeded(_clip_shapes(dict(cfg)), seed, is_clip=True)


def _seeded(shapes: dict, seed: int, is_clip: bool) -> dict[str, torch.Tensor]:
    """fp32 weights, key order fixed: norm weights 1 + 0.1 N, biases 0.02 N, the relative-bias table N(0, 1),
    embeddings N(0, 1) (T5) or 0.02 N (CLIP, as transformers' _init_weights), matrices N(0, fan_in^-1/2)."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for key in sorted(shapes):
        shape = shapes[key]
        r = torch.randn(shape, generator=g)
        if "norm" in key and key.endswith("weight"):
            t = 1.0 + 0.1 * r
        elif key.endswith("bias") and "relative" not in key:
            t = 0.02 * r
        elif "relative_attention_bias" in key:
            t = r
        elif "embedding" in key or key == "shared.weight":
            t = 0.02 * r if is_clip else r
        else:
            t = r * shape[1] ** -0.5
        out[key] = t.contiguous()
    return out


def write_checkpoint(path: str, cfg: dict, weights: dict, fmt: str = "safetensors") -> str:
    os.makedirs(path, exist_ok=True)
    with open(os.path.join(path, "config.json"), "w") as fh:
        json.dump(cfg, fh)
    if fmt == "safetensors":
        from safetensors.torch import save_file

        save_file(weights, os.path.join(path, "model.safetensors"))
    elif fmt == "sharded":
        from safetensors.torch import save_file

        keys = sorted(weights)
        half = len(keys) // 2
        wm = {}
        for i, part in enumerate((keys[:half], keys[half:])):
            name = f"model-{i + 1:05d}-of-00002.safetensors"
            save_file({k: weights[k] for k in part}, os.path.join(path, name))
            wm.update({k: name for k in part})
        with open(os.path.join(path, "model.safetensors.index.json"), "w") as fh:
            json.dump({"metadata": {}, "weight_map": wm}, fh)
    else:
        torch.save(weights, os.path.join(path, "pytorch_model.bin"))
    return path


class ToyTokenizer:
    """Prompts are space-separated integer token ids.  T5 style: ids + [eos], pad 0.  CLIP style: [bos] + ids + [eos],
    padded with pad_token_id.  Truncation keeps the eos, as the HF tokenizers do."""

    def __init__(self, is_clip: bool, bos: int = 0, eos: int = 1, pad: int = 0):
        self.is_clip, self.bos, self.eos, self.pad_token_id = is_clip, bos, eos, pad

    def __call__(self, text, truncation=True, max_length=None, padding="max_length", return_tensors="pt", **_):
        rows = []
        for t in text:
            ids = [int(v) for v in t.split()]
            ids = ([self.bos] if self.is_clip else []) + ids
            ids = ids[: max_length - 1] + [self.eos]
            rows.append(ids + [self.pad_token_id] * (max_length - len(ids)))
        return {"input_ids": torch.tensor(rows, dtype=torch.long)}


def t5_tokenizer():
    return ToyTokenizer(False, eos=1, pad=0)


def clip_tokenizer(eos: int | None = None):
    # legacy rule (config eos_token_id == 2): the tokenizer's eos has the largest id, as in openai/clip-vit-large-patch14
    return ToyTokenizer(True, bos=CLIP_TINY["bos_token_id"], eos=CLIP_TINY["vocab_size"] - 1 if eos is None else eos, pad=1)


def prompts(n: int, lengths, vocab: int, seed: int, avoid=()) -> list[str]:
    g = torch.Generator().manual_seed(seed)
    out = []
    for i in range(n):
        ids = torch.randint(3, vocab - 2, (lengths[i],), generator=g).tolist()
        out.append(" ".join(str(v) for v in ids if v not in avoid))
    return out
