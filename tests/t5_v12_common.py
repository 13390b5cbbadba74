"""Shared pieces of the v1.2 T5 tests (CPU stand-in and GPU): the masked golden of transformers' T5EncoderModel, a toy
tokenizer that returns the attention mask, and one prompt -> latent run of v1.2's inference wiring against the oracle."""
from __future__ import annotations

import os

import numpy as np
import torch

from tests import text_fixtures as tf

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = os.path.join(ROOT, "tests", "golden", "t5_masked.npz")


def golden():
    """(prompts, input_ids [3, 300], attention_mask [3, 300], last_hidden_state [3, 300, 128] fp32)."""
    g = np.load(GOLDEN)
    return ([str(t) for t in g["text"]], torch.from_numpy(g["ids"]), torch.from_numpy(g["mask"]),
            torch.from_numpy(g["out"]))


class MaskingToyTokenizer(tf.ToyTokenizer):
    """The toy T5 tokenizer (ids + eos, pad 0) with the attention mask the HF tokenizers return."""

    def __init__(self):
        super().__init__(False, eos=1, pad=0)

    def __call__(self, text, max_length=None, **kw):
        enc = super().__call__(text, max_length=max_length, **kw)
        enc["attention_mask"] = (enc["input_ids"] != self.pad_token_id).long()
        return enc


def t5_dir(tmp_path, name="google/t5-v1_1-tiny") -> str:
    return tf.write_checkpoint(str(tmp_path / name), tf.T5_TINY, tf.t5_weights(tf.T5_TINY, tf.SEED_T5))


def t5_oracle(ids, mask, dtype=torch.float32):
    """The masked T5 oracle on the tiny golden weights (rounded to bf16 inside when dtype is bf16)."""
    from tests.t5_masked_ref import t5_encode_masked

    return t5_encode_masked(tf.t5_weights(tf.T5_TINY, tf.SEED_T5), tf.T5_TINY, ids, mask, dtype)


def run_pipeline(tmp_path, device: str):
    """v1.2's inference wiring: the "t5" encoder built from its config entry, STDiT3-XS/2 built with the encoder's
    `caption_channels` / `model_max_length`, `t5.y_embedder = model.y_embedder`, then `RFLOW.sample` with the encoded
    prompts, the null caption and the caption mask: three steps, CFG scale 4, the golden's three ragged prompts.
    Oracle: the oracle loop around transformers' fp32 T5 embeddings (the golden) and the fp32 STDiT3 oracle; floor: the
    same loop around the bf16 T5 oracle and the bf16 STDiT3 oracle, latent rounded to bf16 after every step.
    Returns (latent, oracle latent, floor latent, the caption masks the model saw, the prompts' mask)."""
    from opensora.registry import MODELS, build_module
    from opensora.schedulers import RFLOW
    from oracle import sampling_oracle as S, stdit3_oracle as O

    text, ids, mask, hf_out = golden()
    t5 = build_module(dict(type="t5", from_pretrained=t5_dir(tmp_path), model_max_length=300, shardformer=True), MODELS,
                      device=device, tokenizer=MaskingToyTokenizer())
    ocfg = O.STDiT3_XS_2_config(caption_channels=128)
    oracle = O.STDiT3(ocfg).eval()
    O.init_synthetic_weights(oracle, 1234)
    sd = {k: v.to(torch.bfloat16) for k, v in oracle.state_dict().items()}
    oracle.load_state_dict({k: v.float() for k, v in sd.items()})
    oracle = oracle.to(device)
    model = build_module(dict(type="STDiT3-XS/2"), MODELS, caption_channels=t5.output_dim,
                         model_max_length=t5.model_max_length)
    model.load_state_dict(sd)
    model = model.to(device=device, dtype=torch.bfloat16).eval()
    t5.y_embedder = model.y_embedder

    B = len(text)
    g = torch.Generator().manual_seed(77)
    z0 = torch.randn(B, 4, 2, 8, 8, generator=g).to(device=device, dtype=torch.bfloat16)
    extra = {k: torch.full((B,), v, device=device) for k, v in (("fps", 24.0), ("height", 64.0), ("width", 64.0))}
    seen = []
    fwd = model.forward
    model.forward = lambda *a, **k: (seen.append(k.get("mask")), fwd(*a, **k))[1]
    mask_d = mask.to(device)
    with torch.no_grad():
        y = t5.encode(text)
        y_null = t5.null(B)
        assert torch.equal(y["mask"], mask_d) and y["y"].shape == (B, 1, 300, 128)
        out = RFLOW(num_sampling_steps=3, cfg_scale=4.0).sample(model, z0, y["y"], y_null, mask=y["mask"],
                                                                additional_args=extra)
        ref = S.rflow_sample(lambda x, t, y, **kw: oracle(x, t.to(device), y, **kw), z0.float(), hf_out[:, None].to(device),
                             y_null.float(), mask=mask_d, steps=3, cfg_scale=4.0, **extra)
        ob = oracle.to(torch.bfloat16)
        y_bf = t5_oracle(ids, mask, torch.bfloat16)[:, None].float().to(device)
        noise = S.rflow_sample(lambda x, t, y, **kw: ob(x.to(torch.bfloat16).float(), t.to(device), y, **kw).float(),
                               z0.float(), y_bf, y_null.float(), mask=mask_d, steps=3, cfg_scale=4.0, **extra)
    return out, ref, noise, seen, mask_d
