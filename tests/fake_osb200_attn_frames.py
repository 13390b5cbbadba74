"""`attn_frames` entry of the CPU stand-in of the `osb200` binding (TEST INFRASTRUCTURE, not a fallback): a torch
restatement of the osb_attn_frames contract (include/osb200.h) with the kernel's rounding points - fp32 scores, exact
softmax with the row maximum taken over the visible keys, P rounded to bf16 unnormalised before P V, the row sum taken
from the unrounded P, one rounding at the output - and the refusals of the binding and the entry, with the launch-count
convention of tests/fake_osb200.py (one count per launch, nothing counted for a refused call).

`install(monkeypatch)` adds the entry to tests/fake_osb200.py for the duration of one test.  The GPU tests call
`attn_frames` of this module directly on CUDA tensors to pin it to the kernel."""
import torch

from tests import fake_osb200 as base

OsbError = base.OsbError


def install(monkeypatch) -> None:
    monkeypatch.setattr(base, "attn_frames", attn_frames, raising=False)


def visible_keys(Lq: int, Lk: int, frame_tokens: int, q_frame0: int, device) -> torch.Tensor:
    """[Lq] number of keys each query token sees: min(Lk, (q_frame0 + i // frame_tokens + 1) * frame_tokens)."""
    i = torch.arange(Lq, device=device)
    return torch.clamp((q_frame0 + i // frame_tokens + 1) * frame_tokens, max=Lk)


def attn_frames(q, k, v, *, frame_tokens: int, q_frame0: int = 0, out=None, softmax_scale=None):
    for t, n in ((q, "q"), (k, "k"), (v, "v"), (out, "out")):
        base._need(t, torch.bfloat16, n)
    if q.dim() != 3 or k.dim() != 3 or k.shape != v.shape or q.shape[0] != k.shape[0] or q.shape[2] != k.shape[2]:
        raise OsbError(f"attn_frames: q [batch, Lq, D] and k, v [batch, Lk, D] expected, got {tuple(q.shape)}, "
                       f"{tuple(k.shape)}, {tuple(v.shape)}")
    nb, Lq, D = q.shape
    Lk = k.shape[1]
    if out is not None and out.shape != q.shape:
        raise OsbError(f"attn_frames: out must have q's shape {tuple(q.shape)}, got {tuple(out.shape)}")
    if nb > 1 and (k.stride(0) * v.stride(1) != v.stride(0) * k.stride(1)):
        raise OsbError("attn_frames: v must have k's batch stride and out q's (in rows)")
    fail = "osb_attn_frames failed (-1): osb_attn_frames: "
    if D != 512:
        raise OsbError(fail + f"head_dim {D} not built (512)")
    lds = [t.stride(1) if t.shape[1] > 1 else max(t.stride(1), D) for t in (q, k, v)]
    if any(ld < 512 or ld % 8 for ld in lds):
        raise OsbError(fail + "leading dimensions must be >= 512 and multiples of 8")
    if frame_tokens < 1:
        raise OsbError(fail + f"frame_tokens must be >= 1, got {frame_tokens}")
    if Lq < 1:
        raise OsbError(fail + f"empty problem (batch {nb}, Lq {Lq})")
    if q_frame0 < 0 or Lk < 1:
        raise OsbError(fail + f"a query would see no key (q_frame0 {q_frame0}, Lk {Lk})")
    scale = softmax_scale if softmax_scale is not None else D ** -0.5
    sc = (q.float() @ k.float().transpose(1, 2)) * scale
    dead = torch.arange(Lk, device=q.device)[None, :] >= visible_keys(Lq, Lk, frame_tokens, q_frame0, q.device)[:, None]
    sc = sc.masked_fill(dead[None], float("-inf"))
    p = torch.exp(sc - sc.amax(-1, keepdim=True))          # every row sees key 0
    o = ((p.to(torch.bfloat16).float() @ v.float()) / p.sum(-1, keepdim=True)).to(torch.bfloat16)
    base._count("attn_frames", (nb, Lq, Lk, D, frame_tokens, q_frame0))
    if out is None:
        return o
    out.copy_(o)
    return out
