"""Encode time of Open-Sora v1.2's T5 on one GPU: the T5-XXL-shaped encoder (24 x 4096, random weights) at 300 tokens,
batch 1 and 8, with the right-padded attention mask of ragged prompts and without one (the same ids).  Both legs are
warmed up, then timed in alternated windows; the median and the min / max of the per-window means are reported, with
the card name, power limit and max SM clock read in the same run.  Prints one JSON line.

    python tests/t5_v12_bench.py [--iters 10] [--windows 7]"""
import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "open-sora_b200")]

from tests.timing import card, window_ms  # noqa: E402

# prompt lengths in tokens, eos included: one typical prompt, and a batch from the eos-only prompt to a full one
BATCHES = ([40], [1, 17, 40, 60, 77, 120, 200, 300])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--windows", type=int, default=7)
    args = ap.parse_args()
    import osb200
    from opensora.models.text.conditioner import _t5_shapes
    from tests import text_fixtures as tf, text_gpu_common as G

    osb200.init()
    torch.set_grad_enabled(False)
    res = {"gpu": ", ".join(card()), "windows": args.windows, "iters_per_window": args.iters}
    cfg = tf.T5_XXL
    with tempfile.TemporaryDirectory() as tmp:
        w = G.device_weights(_t5_shapes(cfg), False, 1, cfg["d_model"])
        emb = G.build(tmp, cfg, w, False, 300)
        for lens in BATCHES:
            B = len(lens)
            ids = torch.randint(2, cfg["vocab_size"] - 1, (B, 300), device="cuda")
            mask = (torch.arange(300, device="cuda")[None, :] < torch.tensor(lens, device="cuda")[:, None]).long()
            ids[mask == 0] = 0
            legs = {"masked": lambda: emb.encode(ids, mask), "unmasked": lambda: emb.encode(ids)}
            for fn in legs.values():
                window_ms(fn, 3)
            times = {k: [] for k in legs}
            for r in range(args.windows):
                for k in (list(legs) if r % 2 == 0 else list(legs)[::-1]):
                    times[k].append(window_ms(legs[k], args.iters))
            res[f"batch_{B}"] = {"prompt_tokens": lens, **{
                k: {"median_ms": round(statistics.median(v), 3), "min_ms": round(min(v), 3), "max_ms": round(max(v), 3)}
                for k, v in times.items()}}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
