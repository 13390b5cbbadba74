"""Mid-block attention of the causal VAE: the default path (one torch SDPA call per latent frame over the key prefix)
against `osb_attn_frames` (one launch), on the same seeded q / k / v, then the whole decode and encode with
`enable_native_attention()` off and on.  GPU only: without one it fails, it never falls back.

    python tests/vae_attn_bench.py [--out FILE] [--shapes T,h,w ...] [--video T,H,W] [--windows N] [--no-model]

One JSON document: the card's name and power limit read in the same run, and per latent shape (T, h, w) the median and
spread of alternated timing windows after warm-up, algorithmic TFLOP/s from 4 * 512 * hw^2 * T (T + 1) / 2, the peak
of torch.cuda.max_memory_allocated around each path and the rel-L2 between the two outputs at the timed size."""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))

from tests.timing import card, window_ms  # noqa: E402

D = 512


def attention_flop(T: int, hw: int) -> float:
    """QK^T and PV over the visible (query, key) pairs: frame f sees f + 1 frames."""
    return 4.0 * D * hw * hw * T * (T + 1) / 2


def parse(argv=None):
    ap = argparse.ArgumentParser(description=__doc__.split("\n\n")[0])
    triple = lambda s: tuple(int(v) for v in s.split(","))  # noqa: E731
    ap.add_argument("--out", default=None)
    ap.add_argument("--shapes", type=triple, nargs="*", default=[(9, 90, 160), (17, 32, 32), (5, 90, 160)])
    ap.add_argument("--video", type=triple, default=(33, 720, 1280))
    ap.add_argument("--windows", type=int, default=5)
    ap.add_argument("--no-model", action="store_true")
    a = ap.parse_args(argv)
    for s in list(a.shapes) + [a.video]:
        if len(s) != 3 or min(s) < 1:
            ap.error(f"expected T,h,w with positive entries, got {s}")
    return a


def sdpa_loop(q, k, v, T, hw):
    import torch

    o = torch.empty_like(q)
    for f in range(T):
        o[:, :, f * hw:(f + 1) * hw] = torch.nn.functional.scaled_dot_product_attention(
            q[:, :, f * hw:(f + 1) * hw], k[:, :, :(f + 1) * hw], v[:, :, :(f + 1) * hw])
    return o


def bench_shape(T, h, w, windows):
    import osb200
    import torch

    hw = h * w
    g = torch.Generator(device="cuda").manual_seed(T * 1000 + hw)
    q, k, v = ((torch.randn(1, 1, T * hw, D, device="cuda", generator=g)).to(torch.bfloat16) for _ in range(3))
    paths = {"sdpa_loop": lambda: sdpa_loop(q, k, v, T, hw),
             "osb_attn_frames": lambda: osb200.attn_frames(q[:, 0], k[:, 0], v[:, 0], frame_tokens=hw)}
    outs, peak = {}, {}
    for name, fn in paths.items():                      # warm-up, outputs and peak memory
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        outs[name] = fn().reshape(T * hw, D).clone()
        torch.cuda.synchronize()
        peak[name] = (torch.cuda.max_memory_allocated() - base) / 2**20
    one = {n: window_ms(fn, 1) for n, fn in paths.items()}
    reps = {n: max(1, int(300.0 / max(ms, 1e-3))) for n, ms in one.items()}     # ~0.3 s windows
    ms = {n: [] for n in paths}
    for _ in range(windows):                            # alternated windows
        for n, fn in paths.items():
            ms[n].append(window_ms(fn, reps[n]))
    fl = attention_flop(T, hw)
    res = {"latent": [T, h, w], "tokens": T * hw, "tflop": fl / 1e12,
           "rel_l2_between_paths": float((outs["osb_attn_frames"].double() - outs["sdpa_loop"].double()).norm() / outs["sdpa_loop"].double().norm())}
    for n in paths:
        med = statistics.median(ms[n])
        res[n] = {"median_ms": med, "min_ms": min(ms[n]), "max_ms": max(ms[n]), "windows": len(ms[n]), "reps_per_window": reps[n],
                  "tflops": fl / (med * 1e-3) / 1e12, "peak_extra_mib": peak[n]}
    res["speedup"] = res["sdpa_loop"]["median_ms"] / res["osb_attn_frames"]["median_ms"]
    return res


def bench_model(T, H, W):
    import torch
    from opensora.registry import MODELS, build_module

    torch.manual_seed(0)
    with torch.device("cuda"):
        vae = build_module(dict(type="hunyuan_vae"), MODELS, device_map="cuda").eval()
    g = torch.Generator(device="cuda").manual_seed(1)
    lt, lh, lw = vae.get_latent_size([T, H, W])
    z = torch.randn(1, 16, lt, lh, lw, device="cuda", generator=g).to(torch.bfloat16)
    x = (torch.rand(1, 3, T, H, W, device="cuda", generator=g) * 2 - 1).to(torch.bfloat16)
    res = {"video": [T, H, W], "latent": [lt, lh, lw]}
    keep = {}
    with torch.no_grad():
        for leg, fn in (("decode", lambda: vae.decode(z)), ("encode", lambda: vae.encode(x, sample_posterior=False))):
            for native in (False, True):
                (vae.enable_native_attention if native else vae.disable_native_attention)()
                out = fn()                              # warm-up (packs weights)
                del out
                torch.cuda.synchronize()
                torch.cuda.reset_peak_memory_stats()
                # two timed calls of one pass each; the pass's output is kept for the comparison below, and the first
                # call's output stays allocated while the second runs, so the peak covers both
                last = {}
                times = [window_ms(lambda: last.update(out=fn()), 1) for _ in range(2)]
                out = last.pop("out")
                tag = f"{leg}_{'native' if native else 'sdpa'}"
                res[tag] = {"ms": times, "peak_gib": torch.cuda.max_memory_allocated() / 2**30}
                if native:
                    ref = keep.pop(leg).cuda().double()
                    res[f"{leg}_rel_l2_native_vs_sdpa"] = float((out.double() - ref).norm() / ref.norm())
                else:
                    keep[leg] = out.cpu()
                del out
    return res


def main(argv=None):
    a = parse(argv)
    import torch

    if not torch.cuda.is_available():
        raise SystemExit("vae_attn_bench: needs a CUDA device (H100); there is no CPU path for a timing")
    name, q = card()
    if q == "unknown":
        raise SystemExit("vae_attn_bench: nvidia-smi gave no power limit and clock; a timing is not reported without them")
    power, clock = q.split(", ")
    res = {"card": {"name": name, "power_limit": power, "max_sm_clock": clock}, "torch": torch.__version__, "shapes": [],
           "model": None}
    for T, h, w in a.shapes:
        res["shapes"].append(bench_shape(T, h, w, a.windows))
        print(json.dumps(res["shapes"][-1]), flush=True)
    if not a.no_model:
        res["model"] = bench_model(*a.video)
    doc = json.dumps(res, indent=1)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(doc + "\n")
    print(doc)


if __name__ == "__main__":
    main()
