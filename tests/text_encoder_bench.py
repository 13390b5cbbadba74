"""Encode time of text_embedder on one GPU: T5-XXL at B = 2 x 512 tokens and CLIP-L at B = 2 x 77 (random weights),
against the same oracle modules run in bf16 eager torch (cuBLAS) on the same GPU as the library baseline; GEMM TF/s
from osb200's per-launch profile; the card name and power limit read in the same run.  Prints one JSON line.

    python tests/text_encoder_bench.py [--iters 10]"""
import argparse
import json
import os
import sys
import tempfile

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "open-sora_b200")]

from tests.timing import card, window_ms  # noqa: E402


def _time(fn, iters):
    window_ms(fn, 2)   # warm-up
    return window_ms(fn, iters)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    args = ap.parse_args()
    import osb200
    from oracle import text_oracle as O
    from opensora.models.text.conditioner import _clip_shapes, _t5_shapes
    from tests import text_fixtures as tf, text_gpu_common as G

    osb200.init()
    torch.set_grad_enabled(False)
    res = {"gpu": ", ".join(card())}
    with tempfile.TemporaryDirectory() as tmp:
        for tag, cfg, is_clip, L in (("t5_xxl", tf.T5_XXL, False, 512), ("clip_l", tf.CLIP_L, True, 77)):
            shapes = _clip_shapes(cfg) if is_clip else _t5_shapes(cfg)
            w = G.device_weights(shapes, is_clip, 1, cfg["hidden_size" if is_clip else "d_model"])
            emb = G.build(tmp, cfg, w, is_clip, L)
            ids = torch.randint(2, cfg["vocab_size"] - 1, (2, L), device="cuda")
            ms = _time(lambda: emb.encode(ids), args.iters)
            enc = O.clip_encode if is_clip else O.t5_encode
            base = _time(lambda: enc(w, cfg, ids, torch.bfloat16), args.iters)
            osb200.start_profile()
            emb.encode(ids)
            prof = osb200.stop_profile()
            gf = sum(wk for n, wk, _ in prof if n == "gemm")
            gms = sum(t for n, _, t in prof if n == "gemm")
            res[tag] = {"batch": [2, L], "encode_ms": round(ms, 3), "eager_bf16_torch_ms": round(base, 3),
                        "speedup_vs_eager": round(base / ms, 3), "gemm_tflops": round(gf / gms / 1e9, 1),
                        "gemm_share_of_time": round(gms / sum(t for _, _, t in prof), 3)}
            del emb, w
            torch.cuda.empty_cache()
    print(json.dumps(res))


if __name__ == "__main__":
    main()
