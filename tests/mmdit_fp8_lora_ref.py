"""FP8-emulation reference of adapters on the MMDiT FP8 GEMMs (`enable_fp8(..., lora=True)`), for the tests.

On top of tests/mmdit_fp8_ref.py / mmdit_fp8_proj_ref.py, every FP8 Linear whose weight rows belong to an adapted Linear
of `model` computes, for its dequantized e4m3 input x:
    g * (x qdq(W)^T + U bf16(s B)^T) + bias,   U = bf16(x qdq_rows(A)^T)
(the down projection reads the same codes as the base GEMM, with lora_A quantized per row; g is DoRA's column scale, 1
for LoRA).  The reference functions receive weights as slices or concatenations of the state dict's tensors, so each
weight row is traced back to its Linear by its bf16 bit pattern.  `fp8_lora(model)` patches the emulation for the
duration of a `with` block."""
import contextlib

import torch

from tests import fp8_ref as R
from tests import mmdit_fp8_ref as MR


def _row_keys(w: torch.Tensor):
    return [r.tobytes() for r in w.detach().to(torch.bfloat16).contiguous().view(torch.int16).cpu().numpy()]


def _registry(model):
    """{bf16 row bits: (adapter index, row)} and per adapter (A, bf16(s B) as fp32, g or None)."""
    from opensora.utils.lora import _dora_scale, adapter_of, dora_magnitude, is_wrapped

    rows, ads = {}, []
    with torch.no_grad():
        for _, m in model.named_modules():
            if not is_wrapped(m) or adapter_of(m) is None:
                continue
            A, B, s = adapter_of(m)
            g = _dora_scale(m, A, B, s).float() if dora_magnitude(m) is not None else None
            ads.append((A.float(), (s * B.float()).to(torch.bfloat16).float(), g))
            for i, k in enumerate(_row_keys(m.weight)):
                rows[k] = (len(ads) - 1, i)
    return rows, ads


def _lin_with(rows, ads, lin0):
    def lin(x, w, b):
        hits = [rows.get(k) for k in _row_keys(w)]
        if all(h is None for h in hits):
            return lin0(x, w, b)
        base = x @ R.qdq(w.float()).t()
        upd = torch.zeros_like(base)
        g = torch.ones(w.shape[0], dtype=base.dtype, device=base.device)
        for a in sorted({h[0] for h in hits if h is not None}):
            cols = [n for n, h in enumerate(hits) if h is not None and h[0] == a]
            src = [hits[n][1] for n in cols]
            A, sB, ga = (None if t is None else t.to(base.device) for t in ads[a])
            U = (x @ R.qdq(A).t()).to(torch.bfloat16).float()
            upd[..., cols] = U @ sB[src].t()
            if ga is not None:
                g[cols] = ga[src]
        return g * (base + upd) + (0 if b is None else b.float())
    return lin


@contextlib.contextmanager
def fp8_lora(model):
    """Patch the FP8 emulation's GEMM so that the adapters of `model` take part at their FP8 rounding points."""
    rows, ads = _registry(model)
    saved = MR._lin
    MR._lin = _lin_with(rows, ads, saved)
    try:
        yield
    finally:
        MR._lin = saved


def emulation_state(model):
    """The model's bf16 state dict with the adapters' base weights under the plain Linear names (no adapter tensors)."""
    return {k.replace(".base_layer.", "."): v for k, v in model.state_dict().items() if ".lora_" not in k}
