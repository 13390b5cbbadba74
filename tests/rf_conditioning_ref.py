"""Test infrastructure for image / video conditioning (only tests import this module): the fp32 oracle loop of the
conditioned rectified-flow sampler.

Like STDiT3's v1.2 sampler (`oracle/sampling_oracle.py::rflow_sample`) the loop is a restatement of Open-Sora v1.2
`schedulers/rf/__init__.py::RFLOW.sample` (mask branch) and `RFlowScheduler.add_noise`: PARITY UNPINNED, no reference
source or vector exists for it here."""
import torch

from oracle.sampling_oracle import rflow_timestep_transform


def rflow_sample_masked(model, z, y, y_null, frame_mask, noises, mask=None, steps=30, cfg_scale=7.0, transform=None,
                        **model_kw):
    """`rflow_sample` with image / video conditioning.  frame_mask [B, T]: 1 = generate, 0 = keep, in between = edit ratio;
    noises[i] is the noise step i draws.  Per step: x0 = z; upper = frame_mask * 1000 >= t; frames in upper and not yet
    noised become (1 - t/1000) x0 + (t/1000) noise (add_noise); the model sees x_mask = cat[upper, upper]; the Euler update
    is applied to upper frames only, the rest stay x0."""
    B = z.shape[0]
    ts = [(1.0 - i / steps) * 1000.0 for i in range(steps)]
    if transform is not None:
        ts = [rflow_timestep_transform(t, *transform) for t in ts]
    kw = {k: (torch.cat((v, v), 0) if isinstance(v, torch.Tensor) and v.shape[:1] == (B,) else v) for k, v in model_kw.items()}
    if mask is not None:
        kw["mask"] = torch.cat((mask, mask), 0)
    fm = frame_mask.float()
    frames = lambda m: m[:, None, :, None, None]  # noqa: E731
    noise_added = fm == 1
    for i, t in enumerate(ts):
        tv = torch.full((B,), t, dtype=torch.float32, device=z.device)
        x0 = z
        upper = fm * 1000 >= tv[:, None]
        a = tv[:, None, None, None, None] / 1000
        z = torch.where(frames(upper & ~noise_added), (1 - a) * x0 + a * noises[i].float(), x0)
        noise_added = upper
        pred = model(torch.cat((z, z), 0), torch.cat((tv, tv), 0), y=torch.cat((y, y_null), 0), x_mask=upper.repeat(2, 1),
                     **kw).chunk(2, dim=1)[0]
        vc, vu = pred.chunk(2, dim=0)
        t_next = ts[i + 1] if i + 1 < len(ts) else 0.0
        z = z + (vu + cfg_scale * (vc - vu)) * ((t - t_next) / 1000.0)
        z = torch.where(frames(upper), z, x0)
    return z

