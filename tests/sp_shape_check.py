"""Single-GPU kernel parity at the per-rank shapes of the 2-GPU sequence-parallel XL/2 run (debug aid)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))
import torch

from tests.util import cross_case, self_case

for name, fn in (
    ("spatial  B1 T32 S256 H16", lambda: self_case(0, 1, 32, 256, 16, 72)),
    ("temporal B1 T64 S128 H16 (strided view)", lambda: self_case(1, 1, 64, 128, 16, 72)),
    ("temporal B1 T64 S128 H16 (transposed)", lambda: self_case(1, 1, 64, 128, 16, 72, transposed=True)),
    ("temporal B1 T64 S256 H16 (transposed)", lambda: self_case(1, 1, 64, 256, 16, 72, transposed=True)),
    ("cross    N8192 H16", lambda: cross_case(1, 8192, 300, [260], 16)),
    ("cross    N16384 H16", lambda: cross_case(1, 16384, 300, [260], 16)),
):
    try:
        r = fn()
        print(f"{name}: OK {r if r is not None else ''}", flush=True)
    except AssertionError as e:
        print(f"{name}: FAIL {str(e)[:200]}", flush=True)
