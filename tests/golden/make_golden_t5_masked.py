"""Golden of the padding-masked T5 encoder (tests/golden/t5_masked.npz) by EXECUTING transformers' T5EncoderModel in
fp32 with `attention_mask`, as Open-Sora v1.2's T5 wrapper calls it, on the seeded tiny T5 v1.1 checkpoint of
tests/text_fixtures.py (T5_TINY, SEED_T5).

Three prompts of 1 token (eos only), 7 tokens and exactly max_length = 300 tokens (truncated, eos kept), right-padded to
300 by the toy tokenizer (pad 0).  Stored: prompts, input_ids, attention_mask and last_hidden_state.

Run from the repository root: python tests/golden/make_golden_t5_masked.py"""
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))

from tests import text_fixtures as tf  # noqa: E402

MAX_LENGTH = 300


def main():
    from transformers import T5Config, T5EncoderModel

    torch.set_grad_enabled(False)
    text = [""] + tf.prompts(2, (6, 400), tf.T5_TINY["vocab_size"], seed=21)
    ids = tf.t5_tokenizer()(text, max_length=MAX_LENGTH)["input_ids"]
    mask = (ids != 0).long()
    assert mask.sum(1).tolist() == [1, 7, MAX_LENGTH]
    model = T5EncoderModel(T5Config(**tf.T5_TINY)).eval()
    w = tf.t5_weights(tf.T5_TINY, tf.SEED_T5)
    w["encoder.embed_tokens.weight"] = w["shared.weight"]
    model.load_state_dict(w, strict=True)
    out = model(input_ids=ids, attention_mask=mask).last_hidden_state
    dst = os.path.join(ROOT, "tests", "golden", "t5_masked.npz")
    np.savez_compressed(dst, text=np.array(text), ids=ids.numpy(), mask=mask.numpy(), out=out.float().numpy(),
                        t5_cfg=np.array(json.dumps(tf.T5_TINY)), seed=np.array(tf.SEED_T5))
    print("wrote", dst, tuple(out.shape))


if __name__ == "__main__":
    main()
