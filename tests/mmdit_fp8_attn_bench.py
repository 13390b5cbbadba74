"""Measurement of the FP8 attention of MMDiT on one GPU; prints one JSON line.

  python tests/mmdit_fp8_attn_bench.py [--reps 6] [--iters 5] [--no-model]

1. A per-family profile of one bf16 256px forward (bench.py's mmdit leg: B = 3, L = 8 828, C = 3072, 19 + 38 blocks):
   milliseconds, share of the forward and achieved rate of every kernel family (osb200.start_profile).
2. The attention call alone at B = 3, L = 8 828, H = 24, D = 128 (rotate-half RoPE, split QK-norm at token 512):
   osb_attn_short against osb_attn_fp8 (prep included), alternated windows, medians and spreads, TF/s of 4 B L^2 H D
   against the 1 979 TF/s FP8 data-sheet figure (dense, H100 SXM at 700 W), and the rel-L2 of FP8 against bf16.
3. The whole 256px forward in three modes: bf16, FP8 attention, FP8 attention + FP8 MLPs (same model object,
   alternated, median).
The card's name, power limit and max SM clock are read in the same run."""
import argparse
import collections
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.models import B_256PX as B, L_256PX as L, LT_256PX as LT, mmdit_256px  # noqa: E402
from tests.timing import alternate, card, window_ms  # noqa: E402

H, D = 24, 128


def profile(net, inp):
    import osb200

    with torch.no_grad():
        net(**inp)
        torch.cuda.synchronize()
        osb200.start_profile()
        total = window_ms(lambda: net(**inp), 1)
        rec = osb200.stop_profile()
    fam = collections.defaultdict(lambda: [0.0, 0.0, 0])
    for name, work, ms in rec:
        f = fam[name]
        f[0] += ms
        f[1] += work
        f[2] += 1
    out = {"forward_ms_profiled": round(total, 2)}
    for name, (ms, work, n) in sorted(fam.items(), key=lambda kv: -kv[1][0]):
        out[name] = {"ms": round(ms, 2), "share_pct": round(100 * ms / total, 1), "launches": n,
                     "rate_T_per_s": round(work / ms / 1e9, 1)}
    return out


def attention(reps, iters):
    import osb200

    g = torch.Generator(device="cuda").manual_seed(0)
    C = H * D
    qkv = (torch.randn(B * L, 3 * C, device="cuda", generator=g)).to(torch.bfloat16)
    w = [(1 + 0.2 * torch.randn(D, device="cuda", generator=g)).to(torch.bfloat16) for _ in range(4)]
    ang = torch.rand(L, D // 2, device="cuda", generator=g) * 6.28
    kw = dict(num_seqs=B, seqs_per_batch=1, q_strides=(L, 0, 1), k_strides=(L, 0, 1), Lq=L, Lk=L, num_heads=H,
              head_dim=D, q_norm_w=w[0], k_norm_w=w[1], q_norm_w2=w[2], k_norm_w2=w[3], norm_split=LT,
              rope_cos=torch.cos(ang), rope_sin=torch.sin(ang), rope_half=True)
    q, k, v = qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:]
    out_bf, out_f8 = (torch.empty(B * L, C, dtype=torch.bfloat16, device="cuda") for _ in range(2))
    ws = osb200.attn_fp8_workspace(B, L, H, "cuda")
    fns = {"bf16": lambda: osb200.attn_short(q, k, v, out_bf, **kw),
           "fp8": lambda: osb200.attn_fp8(q, k, v, out_f8, workspace=ws, **kw)}
    t = alternate(fns, reps, iters)
    flops = 4.0 * B * L * L * H * D
    res = dict(t)
    for name in ("bf16", "fp8"):
        res[f"{name}_TF_per_s"] = round(flops / t[name] / 1e9, 1)
    res["fp8_TF_per_s_over_1979_datasheet_pct"] = round(100 * res["fp8_TF_per_s"] / 1979.0, 1)
    res["fp8_speedup"] = round(t["bf16"] / t["fp8"], 3)
    res["fp8_vs_bf16_rel_l2"] = float((out_f8.float() - out_bf.float()).norm() / out_bf.float().norm())
    res["fp8_finite"] = bool(torch.isfinite(out_f8).all())
    return res


def model(net, inp, reps):
    modes = {"bf16": (False, False), "fp8_attention": (True, False), "fp8_attention_and_mlps": (True, True)}

    def setmode(m):
        a, mlp = modes[m]
        (net.enable_fp8_attention if a else net.disable_fp8_attention)()
        (net.enable_fp8 if mlp else net.disable_fp8)()

    res, outs = {}, {}
    t = {m: [] for m in modes}
    with torch.no_grad():
        for m in modes:
            setmode(m)
            outs[m] = net(**inp).float()
        for m in ("fp8_attention", "fp8_attention_and_mlps"):
            res[f"{m}_vs_bf16_rel_l2"] = float((outs[m] - outs["bf16"]).norm() / outs["bf16"].norm())
        for i in range(reps):
            for m in (list(modes) if i % 2 == 0 else list(modes)[::-1]):
                setmode(m)
                net(**inp)   # quantizes the weights / warms the workspaces off the clock
                t[m].append(window_ms(lambda: net(**inp), 1))
        setmode("bf16")
    res.update({f"{m}_ms": round(statistics.median(v), 2) for m, v in t.items()})
    res.update({f"{m}_spread_ms": round(max(v) - min(v), 2) for m, v in t.items()})
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=6)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("mmdit_fp8_attn_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power}
    net = inp = None
    if not a.no_model:
        net, inp = mmdit_256px()
        res["bf16_forward_profile"] = profile(net, inp)
    res["attention_B3_L8828_H24"] = attention(a.reps, a.iters)
    if net is not None:
        res["mmdit_256px_forward"] = model(net, inp, a.reps)
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
