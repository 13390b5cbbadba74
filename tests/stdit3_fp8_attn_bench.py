"""Measurement of the FP8 attention of STDiT3 on one GPU; prints one JSON line.

  python tests/stdit3_fp8_attn_bench.py [--reps 5] [--iters 5] [--shapes 64x32x32,32x90x160] [--no-model]

Per latent shape (T x H x W of a [1, 4, T, H, W] latent; STDiT3-XL/2, 16 heads of 72, 300 text tokens):
1. Each attention kind of one block alone: osb_attn_tiles against osb_head_tiles_fp8 + osb_attn_tiles_fp8 (the
   conversion included), and the conversion alone; alternated windows, medians and spreads, and the rate of 4 Lq Lk H D.
2. The attention family's milliseconds per step from osb200.start_profile(), bf16 against FP8 attention (the conversion
   launches reported as their own family).
3. The whole XL/2 step, eager and as a CUDA graph, for bf16, FP8 attention, and FP8 attention + FP8 MLPs (alternated).
The card's name, power limit and max SM clock are read in the same run."""
import argparse
import collections
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.timing import alternate, card  # noqa: E402

H, D, LY = 16, 72, 300


def kinds(T, S, reps, iters):
    """One block's three attentions at T frames of S tokens (batch 1)."""
    import osb200 as osb

    g = torch.Generator(device="cuda").manual_seed(0)
    N = T * S
    res = {}

    def tiles(rows, tmap, nk):
        t = osb.HeadTiles(rows, tmap, nk, H, D, "cuda")
        a = torch.randn(rows, 256, device="cuda", generator=g).to(torch.bfloat16)
        w = (torch.randn(nk * H * D, 256, device="cuda", generator=g) / 16).to(torch.bfloat16)
        osb.gemm_head_tiles(a, w, None, t, nkinds=nk)
        return t

    out = torch.empty(N, H * D, dtype=torch.bfloat16, device="cuda")
    st = tiles(N, osb.tile_map(0, S), 3)
    tt = tiles(N, osb.tile_map(0, T), 3)
    qt = tiles(N, osb.tile_map(0, N, pack=False), 1)
    kv = tiles(LY, osb.tile_map(0, LY, keys_only=True), 2)
    st8, tt8, qt8, kv8 = (osb.HeadTilesFp8(x) for x in (st, tt, qt, kv))
    osb.head_tiles_fp8(kv, kv8, v_period=2, v_slot=1)
    tm_out = osb.tile_map(1, T, S, T)
    calls = {
        "spatial": (4.0 * T * S * S * H * D,
                    lambda: osb.attn_tiles(st, st, out, Lk=S, num_seqs=T),
                    lambda: osb.head_tiles_fp8(st, st8, v_period=3, v_slot=2),
                    lambda: osb.attn_tiles_fp8(st8, st8, out, Lk=S, num_seqs=T)),
        "temporal": (4.0 * S * T * T * H * D,
                     lambda: osb.attn_tiles(tt, tt, out, Lk=T, num_seqs=S, out_map=tm_out),
                     lambda: osb.head_tiles_fp8(tt, tt8, v_period=3, v_slot=2),
                     lambda: osb.attn_tiles_fp8(tt8, tt8, out, Lk=T, num_seqs=S, out_map=tm_out)),
        "cross": (4.0 * N * LY * H * D,
                  lambda: osb.attn_tiles(qt, kv, out, q_kind=0, k_kind=0, v_kind=1, Lk=LY, num_seqs=1),
                  lambda: osb.head_tiles_fp8(qt, qt8),
                  lambda: osb.attn_tiles_fp8(qt8, kv8, out, q_kind=0, k_kind=0, v_kind=1, Lk=LY, num_seqs=1)),
    }
    for name, (work, bf, conv, att) in calls.items():
        t = alternate({"bf16": bf, "fp8": lambda conv=conv, att=att: (conv(), att()), "convert": conv}, reps, iters)
        t["bf16_TF_per_s"] = round(work / t["bf16"] / 1e9, 1)
        t["fp8_TF_per_s"] = round(work / t["fp8"] / 1e9, 1)
        t["speedup"] = round(t["bf16"] / t["fp8"], 3)
        res[name] = t
    return res


def family(net, inp):
    import osb200

    with torch.no_grad():
        net(**inp)
        torch.cuda.synchronize()
        osb200.start_profile()
        net(**inp)
        rec = osb200.stop_profile()
    fam = collections.defaultdict(lambda: [0.0, 0])
    for name, _, ms in rec:
        fam[name][0] += ms
        fam[name][1] += 1
    return {k: {"ms": round(v[0], 2), "launches": v[1]} for k, v in fam.items() if "attn" in k or "tiles" in k}


def model(T, Hx, Wx, reps, iters, graphs):
    from opensora.models.stdit.stdit3 import STDiT3_XL_2

    torch.manual_seed(0)
    net = STDiT3_XL_2().to("cuda", torch.bfloat16).eval()
    inp = dict(x=torch.randn(1, 4, T, Hx, Wx, device="cuda"), timestep=torch.tensor([500.0], device="cuda"),
               y=torch.randn(1, 1, LY, 4096, device="cuda"), mask=torch.ones(1, LY, dtype=torch.int32, device="cuda"),
               fps=torch.tensor([24.0], device="cuda"), height=[Hx * 8], width=[Wx * 8])
    modes = {"bf16": (False, False), "fp8_attn": (True, False), "fp8_attn_mlp": (True, True)}

    def setmode(a, m):
        (net.enable_fp8_attention if a else net.disable_fp8_attention)()
        (net.enable_fp8 if m else net.disable_fp8)()

    res = {"family": {}}
    for k, (a, m) in modes.items():
        setmode(a, m)
        res["family"][k] = family(net, inp)
    setmode(True, True)

    def eager(a, m):
        def f():   # the switches alone: the FP8 weights and tile workspaces stay cached across the windows
            net._fp8_attn, net._fp8 = a, m
            with torch.no_grad():
                net(**inp)
        return f

    res["eager_ms"] = alternate({k: eager(*v) for k, v in modes.items()}, reps, iters)
    if graphs:
        replays = {}
        for k, (a, m) in modes.items():
            net._fp8_attn, net._fp8 = a, m
            replays[k] = net.capture(**inp)
        res["graph_ms"] = alternate({k: (lambda r=r: r.graph.replay()) for k, r in replays.items()}, reps, iters)
        del replays
    setmode(False, False)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--iters", type=int, default=5)
    ap.add_argument("--shapes", default="64x32x32,32x90x160")
    ap.add_argument("--no-model", action="store_true")
    ap.add_argument("--no-graphs", action="store_true")
    a = ap.parse_args()
    import osb200

    osb200.init(0)
    name, q = card()
    out = {"card": name, "power_limit_and_max_sm_clock": q}
    for shape in a.shapes.split(","):
        T, Hx, Wx = (int(v) for v in shape.split("x"))
        S = (Hx // 2) * (Wx // 2)
        r = {"kinds": kinds(T, S, a.reps, 20)}
        if not a.no_model:
            r["model"] = model(T, Hx, Wx, a.reps, a.iters, not a.no_graphs)
        out[shape] = r
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
