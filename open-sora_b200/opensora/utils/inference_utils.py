"""Image / video conditioning of STDiT3 by mask strategy, in latent space: Open-Sora v1.2 `opensora/utils/inference_utils.py`
(`parse_mask_strategy`, `find_nearest_point`, `apply_mask_strategy`, `append_generated`), the helpers the reference's
`gradio/app.py:191-207` imports and drives at `:285-298` (image prompt -> strategy "0"), `:406` (apply, align=5) and
`:398-402,437-476` (multi-clip loop).  Absent from the reference tree like STDiT3 itself: restated, **parity unpinned**.

A mask strategy is a `;`-separated list of entries `loop_id,ref_id,ref_start,target_start,length,edit_ratio`: in loop
`loop_id`, frames [ref_start, ref_start + length) of the sample's reference `ref_id` are written into the latent at
target_start and kept (edit_ratio 0) or re-generated from a partly noised copy (0 < edit_ratio < 1) by
`RFLOW.sample(frame_mask=...)`.  References are latents: `refs_x[b]` is a list of [C, T, H, W] tensors (or None)."""
from __future__ import annotations

import torch

MASK_DEFAULT = ["0", "0", "0", "0", "1", "0"]


def parse_mask_strategy(mask_strategy: str | None) -> list[list]:
    """"0,0,0,0,1,0;1,0,-5" -> [[0, 0, 0, 0, 1, 0.0], [1, 0, -5, 0, 1, 0.0]]: missing trailing fields take MASK_DEFAULT,
    the first five are ints, the edit ratio a float.  None or "" -> []."""
    out = []
    if not mask_strategy:
        return out
    for entry in mask_strategy.split(";"):
        fields = entry.split(",")
        if not 1 <= len(fields) <= 6:
            raise ValueError(f"invalid mask strategy entry {entry!r}: 1 to 6 comma-separated fields")
        fields = fields + MASK_DEFAULT[len(fields):]
        out.append([int(f) for f in fields[:5]] + [float(fields[5])])
    return out


def find_nearest_point(value: int, point: int, max_value: int) -> int:
    """Snap `value` to a multiple of `point`: down, or up when past the half way and the next multiple stays below the last
    whole block of `max_value`."""
    t = value // point
    if value % point > point / 2 and t < max_value // point - 1:
        t += 1
    return t * point


def apply_mask_strategy(z: torch.Tensor, refs_x, mask_strategys, loop_i: int, align: int | None = None):
    """Write the reference latents the strategies name for loop `loop_i` into z [B, C, T, H, W] (in place) and return the
    frame mask fp32 [B, T] (1 where no entry applies, the entry's edit ratio where one does), or None for an empty list."""
    if len(mask_strategys) == 0:
        return None
    T = z.shape[2]
    masks = []
    for i, strategy in enumerate(mask_strategys):
        mask = torch.ones(T, dtype=torch.float32, device=z.device)
        for loop_id, ref_id, ref_start, target_start, length, edit_ratio in parse_mask_strategy(strategy):
            if loop_id != loop_i:
                continue
            ref = refs_x[i][ref_id]                       # [C, T_ref, H, W]
            if ref_start < 0:
                ref_start += ref.shape[1]
            if target_start < 0:
                target_start += T
            if align is not None:
                ref_start = find_nearest_point(ref_start, align, ref.shape[1])
                target_start = find_nearest_point(target_start, align, T)
            length = min(length, T - target_start, ref.shape[1] - ref_start)
            z[i, :, target_start:target_start + length] = ref[:, ref_start:ref_start + length]
            mask[target_start:target_start + length] = edit_ratio
        masks.append(mask)
    return torch.stack(masks)


def append_generated(vae, generated, refs_x, mask_strategy, loop_i: int, condition_frame_length: int,
                     condition_frame_edit: float, is_latent: bool = False):
    """Make the clip just generated a reference of loop `loop_i`: its last `condition_frame_length` latent frames become the
    first ones of the next clip (edit ratio `condition_frame_edit`).  `generated` [B, C, T, H, W] is encoded with `vae` unless
    `is_latent`.  Updates and returns (refs_x, mask_strategy)."""
    ref_x = generated if is_latent else vae.encode(generated)
    for j in range(len(refs_x)):
        if refs_x[j] is None:
            refs_x[j] = [ref_x[j]]
        else:
            refs_x[j].append(ref_x[j])
        mask_strategy[j] = "" if not mask_strategy[j] else mask_strategy[j] + ";"
        L = condition_frame_length
        mask_strategy[j] += f"{loop_i},{len(refs_x[j]) - 1},-{L},0,{L},{condition_frame_edit}"
    return refs_x, mask_strategy


def sample_looped(scheduler, model, shape, y, y_null, refs_x, mask_strategy, num_loop: int, condition_frame_length: int,
                  condition_frame_edit: float = 0.0, *, align: int | None = None, generator: torch.Generator | None = None,
                  device=None, dtype=torch.bfloat16, **sample_kw) -> torch.Tensor:
    """Long video in `num_loop` clips (gradio/app.py:394-402,469-472, in latent space): loop i draws z `shape` [B, C, T, H, W]
    from `generator`, applies the strategies and samples it with `scheduler.sample(model, z, y, y_null, frame_mask=...)`;
    from loop 1 on, the previous clip is first appended as a reference (`append_generated`), so that clip i starts with the
    last `condition_frame_length` latent frames of clip i - 1.  Returns clip 0 followed by every later clip without those
    first frames, concatenated along T.  `refs_x` / `mask_strategy` (one entry per sample) are updated in place."""
    clips = []
    for loop_i in range(num_loop):
        if loop_i > 0:
            append_generated(None, clips[-1], refs_x, mask_strategy, loop_i, condition_frame_length, condition_frame_edit,
                             is_latent=True)
        z = torch.randn(shape, generator=generator, device=device, dtype=dtype)
        frame_mask = apply_mask_strategy(z, refs_x, mask_strategy, loop_i, align=align)
        clips.append(scheduler.sample(model, z, y, y_null, frame_mask=frame_mask, generator=generator, **sample_kw))
    return torch.cat([clips[0]] + [c[:, :, condition_frame_length:] for c in clips[1:]], dim=2)
