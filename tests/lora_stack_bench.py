"""Measurement of stacked LoRA / DoRA adapters on one GPU; prints one JSON line.

  python tests/lora_stack_bench.py [--reps 5]

The whole MMDiT 256px forward (bench.py's mmdit leg: B = 3) with adapters on every block Linear, in four states put on
and taken off the same model object:
  plain            no adapter;
  one_r64          one LoRA adapter of rank 64;
  two_r32          two LoRA adapters of rank 32;
  lora_dora_lora   LoRA r = 16, DoRA r = 32, LoRA r = 16, in that order.
The three adapted states have the same total rank, so their packs have the same shapes (A_cat [64, K]) and their
forwards the same launches; the DoRA state also moves the modulation layers out of the grouped GEMM, as one DoRA
adapter does.  Median and spread of --reps windows of one forward each, the order of the states reversed every other
round.  The card's name and power limit are read in the same run."""
import argparse
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "open-sora_b200")):
    if p not in sys.path:
        sys.path.insert(0, p)

from tests.models import mmdit_256px  # noqa: E402
from tests.timing import card, window_ms  # noqa: E402

# state -> [(rank, DoRA)] in the order the forward applies them
STATES = {"plain": [], "one_r64": [(64, False)], "two_r32": [(32, False), (32, False)],
          "lora_dora_lora": [(16, False), (32, True), (16, False)]}


def _wrap(lin, spec):
    from opensora.utils.lora import LoraLinear

    w = None
    for k, (r, dora) in enumerate(spec):
        name = f"a{k}"
        if w is None:
            w = LoraLinear(lin, r, 1.0, use_dora=dora, adapter_name=name)
        else:
            w.add_adapter(name, r, 1.0, use_dora=dora)
        torch.nn.init.normal_(w.lora_A[name].weight, std=lin.in_features ** -0.5)
        torch.nn.init.normal_(w.lora_B[name].weight, std=1e-3)
        if dora:
            w.lora_magnitude_vector[name].weight.copy_(lin.weight.float().norm(dim=1) * 1.1)
    w.active_adapters = [f"a{k}" for k in range(len(spec))]
    return w


def model(reps):
    import osb200

    net, inp = mmdit_256px()
    res = {}
    with torch.no_grad():
        sites = []
        for blocks in (net.double_blocks, net.single_blocks):
            for name, lin in list(blocks.named_modules()):
                if type(lin) is torch.nn.Linear:
                    parent, _, attr = name.rpartition(".")
                    sites.append((blocks.get_submodule(parent) if parent else blocks, attr, lin,
                                  {k: _wrap(lin, spec) if spec else lin for k, spec in STATES.items()}))
        res["adapted_linears"] = len(sites)

        def put(state: str):
            for parent, attr, _, alts in sites:
                setattr(parent, attr, alts[state])
            net._drop_caches()

        for k in STATES:
            put(k)
            out = net(**inp)   # builds the packs (and DoRA's g) off the clock
            l0 = osb200.launch_count()
            net(**inp)
            res[f"launches_{k}"] = osb200.launch_count() - l0
            res[f"finite_{k}"] = bool(torch.isfinite(out).all())
        t = {k: [] for k in STATES}
        for i in range(reps):
            for k in (list(STATES) if i % 2 == 0 else list(STATES)[::-1]):
                put(k)
                net(**inp)   # re-reads the cached packs after the swap (off the clock)
                t[k].append(window_ms(lambda: net(**inp), 1))
        put("plain")
    res.update({f"{k}_ms": round(statistics.median(v), 2) for k, v in t.items()})
    res.update({f"{k}_spread_ms": round(max(v) - min(v), 2) for k, v in t.items()})
    for k in ("two_r32", "lora_dora_lora"):
        res[f"{k}_over_one_r64_pct"] = round(100.0 * (res[f"{k}_ms"] / res["one_r64_ms"] - 1.0), 2)
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=5)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("lora_stack_bench.py measures on a CUDA device (H100); there is nothing to measure without one")
    import osb200

    osb200.init(0)
    name, power = card()
    res = {"card": name, "power_limit,max_sm_clock": power, "mmdit_256px_forward": model(a.reps)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
