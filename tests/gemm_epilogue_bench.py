"""Per-shape cost of the bf16 GEMM epilogues at the STDiT3-XL/2 benchmark shape; prints one JSON line.

  python tests/gemm_epilogue_bench.py [--reps 7] [--iters 20]

The six GEMMs of one STDiT3 block at M = 16 384 token rows (latent 64x32x32, C = 1152, 16 heads of 72):
  qkv        1152 -> 3456  head tiles (spatial map, RMSNorm on q and k)
  proj       1152 -> 1152  bias, gate, residual, in place (out = residual)
  cross_q    1152 -> 1152  head tiles (one kind)
  cross_proj 1152 -> 1152  bias, residual, in place
  fc1        1152 -> 4608  bias, GELU-tanh
  fc2        4608 -> 1152  bias, gate, residual, in place
Each is timed with its production epilogue ("epi") and as a plain EPI_BIAS GEMM of the same shape into a separate output
("bias"), alternated in the same loop: median and spread of --reps windows of --iters calls, CUDA events.  epi - bias is
what the epilogue costs on top of the main loop.  `per_step_ms` scales by the 28 spatial + 28 temporal blocks of a step.
The card's name and power limit are read in the same run."""
import argparse
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.timing import alternate, card  # noqa: E402

M_ROWS, C, HEADS, HEAD_DIM, S = 16384, 1152, 16, 72, 256
BLOCKS = 56
SHAPES = {"qkv": (C, 3 * C), "proj": (C, C), "cross_q": (C, C), "cross_proj": (C, C), "fc1": (C, 4 * C),
          "fc2": (4 * C, C)}


def epilogue_calls():
    """name -> (production call, EPI_BIAS call of the same shape, K, N)."""
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    rn = lambda *s, sc=1.0: (torch.randn(*s, device="cuda", generator=g) * sc).to(torch.bfloat16)   # noqa: E731
    calls = {}
    for name, (K, N) in SHAPES.items():
        x, w, b = rn(M_ROWS, K), rn(N, K, sc=K ** -0.5), rn(N, sc=0.1)
        out = torch.empty(M_ROWS, N, dtype=torch.bfloat16, device="cuda")
        bias_only = (lambda x=x, w=w, b=b, out=out: osb200.gemm(x, w, b, out=out))
        if name in ("qkv", "cross_q"):
            if name == "qkv":
                tiles = osb200.HeadTiles(M_ROWS, osb200.tile_map(0, S), 3, HEADS, HEAD_DIM, "cuda")
                norm = (rn(HEAD_DIM), rn(HEAD_DIM), None)
                prod = (lambda x=x, w=w, b=b, t=tiles, nw=norm: osb200.gemm_head_tiles(x, w, b, t, nkinds=3, norm_w=nw))
            else:
                tiles = osb200.HeadTiles(M_ROWS, osb200.tile_map(0, M_ROWS, pack=False), 1, HEADS, HEAD_DIM, "cuda")
                prod = (lambda x=x, w=w, b=b, t=tiles: osb200.gemm_head_tiles(x, w, b, t, nkinds=1))
        elif name == "fc1":
            prod = (lambda x=x, w=w, b=b, out=out: osb200.gemm(x, w, b, epilogue=osb200.EPI_BIAS_GELU_TANH, out=out))
        else:
            # the residual stream xs is updated in place; the adaLN table of one sample is [1, 6, C], gate = m[:, k]
            xs = rn(M_ROWS, N)
            m = torch.randn(1, 6, N, device="cuda", generator=g) * 0.1
            gate = None if name == "cross_proj" else m[:, 2]
            prod = (lambda x=x, w=w, b=b, xs=xs, gate=gate: osb200.gemm(
                x, w, b, epilogue=osb200.EPI_BIAS_GATE_RES, residual=xs, gate=gate, group_rows=M_ROWS, out=xs))
        calls[name] = (prod, bias_only, K, N)
    return calls


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=7)
    ap.add_argument("--iters", type=int, default=20)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("gemm_epilogue_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "rows": M_ROWS, "gemm_ms": {}}
    total_epi = total_cost = 0.0
    for k, (prod, bias_only, K, N) in epilogue_calls().items():
        t = alternate({"epi": prod, "bias": bias_only}, a.reps, a.iters, warmup=3)
        t["epi_cost"] = round(t["epi"] - t["bias"], 4)
        flop = 2.0 * M_ROWS * N * K
        t["epi_tflops"] = round(flop / (t["epi"] * 1e-3) / 1e12, 1)
        t["bias_tflops"] = round(flop / (t["bias"] * 1e-3) / 1e12, 1)
        res["gemm_ms"][k] = t
        total_epi += t["epi"]
        total_cost += t["epi_cost"]
    res["per_step_ms"] = {"six_gemms": round(BLOCKS * total_epi, 2), "epilogue_cost": round(BLOCKS * total_cost, 2)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
