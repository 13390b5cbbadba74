"""The rectified-flow sampling loop that drives STDiT3 (Open-Sora v1.2 `opensora/schedulers/rf/__init__.py::RFLOW.sample`
+ `rectified_flow.py::timestep_transform`).  Like STDiT3 itself it is ABSENT from the reference tree (v2.0.0 ships the
MMDiT sampler, mirrored in `opensora/utils/sampling.py`); this is the restatement of SURVEY.md Appendix A, row "RF sampler" -
**parity unpinned**, self-consistent with `oracle/sampling_oracle.py::rflow_sample`.

Per step: the latent is doubled (conditional | null-caption branch, "CFG batch 2"), the model predicts a velocity (its first
`out_channels / 2` channels when `pred_sigma`), `v = v_u + s (v_c - v_u)`, `z += v * (t_i - t_{i+1}) / 1000`.  The combine +
Euler update is ONE `osb_cfg_euler` launch (two-branch mode).

Image / video conditioning (v1.2 `mask` argument, here `frame_mask` [B, T]: 1 = generate, 0 = keep the reference written into
`z`, in between = edit ratio; built by `opensora.utils.inference_utils.apply_mask_strategy`), also restated and **parity
unpinned** (self-consistent with `tests/rf_conditioning_ref.py::rflow_sample_masked`).  Frame f of sample b takes part in step i
when `frame_mask * 1000 >= t_i` (the model gets that as `x_mask`, so kept frames are modulated with timestep 0); other frames
keep their values bit for bit.  A frame with edit ratio e stays the reference while t > e * 1000 and is re-noised once, at
the first t_i <= e * 1000, to (1 - t_i/1000) z + (t_i/1000) noise (SDEdit).  One noise tensor is drawn per step, as upstream's
`randn_like`.  Each step's update and the next step's re-noise are ONE `osb_rf_masked_step` launch (plus one re-noise-only
launch before the first step); the schedule stays on the device, so the loop never synchronises with the host."""
from __future__ import annotations

import torch

from opensora.registry import SCHEDULERS


def timestep_transform(t: torch.Tensor, height, width, num_frames, base_resolution: int = 512 * 512, base_num_frames: int = 1,
                       scale: float = 1.0, num_timesteps: int = 1000) -> torch.Tensor:
    """Resolution- and length-aware shift of the schedule: t' = r t / (1 + (r - 1) t) on t in [0, 1] with
    r = sqrt(H W / 512^2) * sqrt(frames // 17 * 5) (videos; 1 for images) * scale."""
    t = t / num_timesteps
    ratio_space = (torch.as_tensor(height, dtype=torch.float32) * torch.as_tensor(width, dtype=torch.float32) / base_resolution).sqrt()
    frames = torch.as_tensor(num_frames)
    eff = torch.ones_like(frames, dtype=torch.float32) if int(frames.reshape(-1)[0]) == 1 else (frames // 17 * 5).float()
    ratio = ratio_space * (eff / base_num_frames).sqrt() * scale
    return ratio * t / (1 + (ratio - 1) * t) * num_timesteps


@SCHEDULERS.register_module("rflow")
class RFLOW:
    def __init__(self, num_sampling_steps: int = 30, num_timesteps: int = 1000, cfg_scale: float = 7.0,
                 use_timestep_transform: bool = False, **kwargs):
        self.num_sampling_steps, self.num_timesteps = num_sampling_steps, num_timesteps
        self.cfg_scale, self.use_timestep_transform = cfg_scale, use_timestep_transform

    def schedule(self, batch: int, device, additional_args: dict | None = None) -> list[torch.Tensor]:
        """Descending timesteps [B] per step: (1 - i / N) * 1000, optionally transformed per sample."""
        ts = [(1.0 - i / self.num_sampling_steps) * self.num_timesteps for i in range(self.num_sampling_steps)]
        ts = [torch.full((batch,), t, device=device, dtype=torch.float32) for t in ts]
        if self.use_timestep_transform:
            a = additional_args or {}
            ts = [timestep_transform(t, a["height"].to(device), a["width"].to(device), a["num_frames"].to(device),
                                     num_timesteps=self.num_timesteps) for t in ts]
        return ts

    def sample(self, model, z: torch.Tensor, y: torch.Tensor, y_null: torch.Tensor, mask=None, additional_args: dict | None = None,
               guidance_scale: float | None = None, progress: bool = False, frame_mask: torch.Tensor | None = None,
               generator: torch.Generator | None = None) -> torch.Tensor:
        """z [B, C, T, H, W] noise (bf16 on the model's device), y [B, 1, L, D] caption embeddings, y_null the null caption
        (`model.y_embedder.y_embedding` broadcast, as upstream's `text_encoder.null`), mask [B, L] caption mask.  Extra model
        inputs (fps, height, width, num_frames) ride in `additional_args`.  Returns the denoised latent.
        frame_mask [B, T] (upstream's `mask`): conditioned sampling, see the module docstring; the reference latents must
        already be in `z`.  `generator` draws its per-step noise (default: torch's global generator for z's device)."""
        import osb200

        s = self.cfg_scale if guidance_scale is None else guidance_scale
        B = z.shape[0]
        kw = dict(additional_args or {})
        kw.pop("num_frames", None)            # consumed by the schedule, not a model input
        args = {k: (torch.cat((v, v), 0) if isinstance(v, torch.Tensor) and v.shape[:1] == (B,) else v) for k, v in kw.items()}
        args["y"] = torch.cat((y, y_null), 0)
        if mask is not None:
            args["mask"] = torch.cat((mask, mask), 0)   # upstream passes the caption mask unchanged to both branches
        ts = self.schedule(B, z.device, additional_args)
        z = z.contiguous()
        if frame_mask is not None:
            return self._sample_masked(osb200, model, z, args, ts, frame_mask, float(s), generator)
        for i, t in enumerate(ts):
            pred = model(torch.cat((z, z), 0), torch.cat((t, t), 0), **args)
            pred = pred.chunk(2, dim=1)[0]                                   # drop the sigma half (pred_sigma)
            vc, vu = (p.to(z.dtype).contiguous() for p in pred.chunk(2, dim=0))
            t_next = ts[i + 1] if i + 1 < len(ts) else torch.zeros_like(t)
            dt = (t - t_next) / self.num_timesteps
            if bool((dt != dt[0]).any()):     # per-sample step sizes (different resolutions in one batch): one launch per sample
                z = torch.cat([osb200.cfg_euler(vc[b:b + 1], vu[b:b + 1], None, z[b:b + 1], g_txt=float(s), dt=float(dt[b]))
                               for b in range(B)], 0)
            else:
                z = osb200.cfg_euler(vc, vu, None, z, g_txt=float(s), dt=float(dt[0]))
        return z

    def _sample_masked(self, osb200, model, z, args, ts, frame_mask, s, generator):
        N = self.num_timesteps
        fm = frame_mask.to(device=z.device, dtype=torch.float32).contiguous()
        sched = torch.stack(ts + [torch.zeros_like(ts[0])]).contiguous()      # [steps + 1, B] on the device, t_n = 0

        def randn():
            return torch.randn(z.shape, generator=generator, device=z.device, dtype=z.dtype)

        # step 0's re-noise (frames with 0 < edit ratio whose t_0 is already reached); then each launch ends step i and
        # starts step i + 1 with the noise step i + 1 draws
        z = osb200.rf_masked_step(None, None, z, fm, sched[0], sched[0], guidance=s, noise=randn(), update=False,
                                  num_timesteps=N)
        for i in range(len(ts)):
            t = sched[i]
            args["x_mask"] = (fm * N >= t[:, None]).repeat(2, 1)
            pred = model(torch.cat((z, z), 0), torch.cat((t, t), 0), **args)
            pred = pred.chunk(2, dim=1)[0]
            vc, vu = (p.to(z.dtype).contiguous() for p in pred.chunk(2, dim=0))
            noise = randn() if i + 1 < len(ts) else None
            osb200.rf_masked_step(vc, vu, z, fm, sched[i], sched[i + 1], guidance=s, noise=noise, num_timesteps=N, out=z)
        return z
