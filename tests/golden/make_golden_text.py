"""Goldens of the text encoders (tests/golden/text_encoders.npz) by EXECUTING the reference's own `HFEmbedder`
(opensora/models/text/conditioner.py:10-53, shardformer=False) on transformers' T5EncoderModel / CLIPTextModel, loaded
from seeded toy checkpoints (tests/text_fixtures.py).  ColossalAI and the shardformer policy are stubbed (never called
with shardformer=False); the tokenizer classes return the toy tokenizer, whose ids are stored with the outputs.

Stored: seeds, configs, token ids and fp32 outputs of
  - tiny T5 (gated-gelu, d_kv 64, 2 heads, 2 layers) at max_length 512, and with added_tokens=5, seq_align=16;
  - tiny CLIP (2 layers, 77 tokens) under both pooling rules (legacy eos_token_id == 2: argmax; else first eos);
  - transformers' T5 bucket of every relative offset -1023..1023 (bidirectional, 32 buckets, max_distance 128).

Run from the repository root: python tests/golden/make_golden_text.py"""
import json
import os
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))

from oracle import ref_loader  # noqa: E402
from tests import text_fixtures as tf  # noqa: E402


def load_reference_conditioner():
    """The reference's conditioner.py with colossalai, the T5 shardformer policy and the registry stubbed."""
    saved = {k: v for k, v in sys.modules.items() if k == "opensora" or k.startswith("opensora.")}
    for k in saved:
        del sys.modules[k]
    try:
        for pkg in ("opensora", "opensora.models", "opensora.models.text", "opensora.acceleration",
                    "opensora.acceleration.shardformer", "opensora.acceleration.shardformer.policy", "colossalai"):
            ref_loader._shell(pkg)
        sf = types.ModuleType("colossalai.shardformer")
        sf.ShardConfig = sf.ShardFormer = None
        sys.modules["colossalai.shardformer"] = sf
        pol = types.ModuleType("opensora.acceleration.shardformer.policy.t5_encoder")
        pol.T5EncoderPolicy = None
        sys.modules["opensora.acceleration.shardformer.policy.t5_encoder"] = pol
        reg = types.ModuleType("opensora.registry")

        class _R:
            def register_module(self, *a, **k):
                return lambda f: f

        reg.MODELS = _R()
        sys.modules["opensora.registry"] = reg
        return ref_loader._load("opensora.models.text.conditioner",
                                os.path.join(ref_loader.REF, "opensora", "models", "text", "conditioner.py"))
    finally:
        for k in [k for k in sys.modules if k == "opensora" or k.startswith("opensora.")]:
            del sys.modules[k]
        sys.modules.update(saved)


def _toy(tok):
    class _Tok:
        @staticmethod
        def from_pretrained(*a, **k):
            return tok
    return _Tok


def main():
    torch.set_grad_enabled(False)
    cond = load_reference_conditioner()
    out = {}
    with tempfile.TemporaryDirectory() as tmp:
        # ---- T5 ----
        t5_dir = tf.write_checkpoint(os.path.join(tmp, "google", "t5-tiny"), tf.T5_TINY, tf.t5_weights(tf.T5_TINY, tf.SEED_T5))
        cond.T5Tokenizer = _toy(tf.t5_tokenizer())
        emb = cond.HFEmbedder(t5_dir, max_length=512, shardformer=False)
        ids_seen = []
        fwd = emb.hf_module.forward
        emb.hf_module.forward = lambda input_ids=None, **k: (ids_seen.append(input_ids.clone()), fwd(input_ids=input_ids, **k))[1]
        text = tf.prompts(2, (40, 700), tf.T5_TINY["vocab_size"], seed=7)
        out["t5_out"] = emb(text).float().numpy()
        out["t5_ids"] = ids_seen[-1].numpy()
        out["t5_pad_out"] = emb(text, added_tokens=5, seq_align=16).float().numpy()
        out["t5_pad_ids"] = ids_seen[-1].numpy()
        out["t5_text"] = np.array(text)
        # ---- CLIP, both pooling rules ----
        for tag, cfg, tok in (("legacy", tf.CLIP_TINY, tf.clip_tokenizer()),
                              ("eos", dict(tf.CLIP_TINY, eos_token_id=300), tf.clip_tokenizer(eos=300))):
            d = tf.write_checkpoint(os.path.join(tmp, "openai", f"clip-tiny-{tag}"), cfg, tf.clip_weights(cfg, tf.SEED_CLIP))
            cond.CLIPTokenizer = _toy(tok)
            emb = cond.HFEmbedder(d, max_length=77)
            ids_seen = []
            fwd = emb.hf_module.forward
            emb.hf_module.forward = lambda input_ids=None, _f=fwd, **k: (ids_seen.append(input_ids.clone()), _f(input_ids=input_ids, **k))[1]
            text = tf.prompts(3, (10, 30, 120), cfg["vocab_size"], seed=11, avoid=(300,))
            out[f"clip_{tag}_out"] = emb(text).float().numpy()
            out[f"clip_{tag}_ids"] = ids_seen[-1].numpy()
            out[f"clip_{tag}_cfg"] = np.array(json.dumps(cfg))
    from transformers.models.t5.modeling_t5 import T5Attention

    rel = torch.arange(-1023, 1024)
    out["t5_buckets"] = T5Attention._relative_position_bucket(rel, bidirectional=True, num_buckets=32, max_distance=128).numpy()
    out["t5_cfg"] = np.array(json.dumps(tf.T5_TINY))
    out["seeds"] = np.array([tf.SEED_T5, tf.SEED_CLIP])
    dst = os.path.join(ROOT, "tests", "golden", "text_encoders.npz")
    np.savez_compressed(dst, **out)
    print("wrote", dst, {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    main()
