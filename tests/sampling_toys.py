"""Deterministic stand-ins for the four models `prepare_api` drives (denoiser, autoencoder, T5, CLIP): small closed-form
functions that depend on EVERY input the pipeline hands them, so a wrong tensor anywhere changes the result.  Shared by
tests/golden/make_golden_sampling.py (which runs the REFERENCE's `prepare_api` on them) and tests/test_sampling_cpu.py
(which runs ours)."""
import torch
import torch.nn as nn


class ToyDenoiser(nn.Module):
    def __init__(self):
        super().__init__()
        self.w = nn.Parameter(torch.tensor(0.7))
        self.seen = []

    def forward(self, img, img_ids, txt, txt_ids, timesteps, y_vec, cond=None, guidance=None, **kw):
        self.seen.append(sorted(kw))
        f = img.float()
        pos = (img_ids.float() * torch.tensor([0.01, 0.003, 0.002])).sum(-1, keepdim=True)
        c = 0.0 if cond is None else cond.float()[..., : f.shape[-1]] * 0.3
        t = txt.float().mean(dim=(1, 2))[:, None, None] + txt_ids.float().sum(dim=(1, 2))[:, None, None]
        y = y_vec.float().mean(-1)[:, None, None]
        r = torch.tanh(f * self.w.float() + c + pos) * (1 + timesteps.float()[:, None, None]) + 0.2 * t + 0.1 * y
        return (r + 0.01 * guidance.float()[:, None, None]).to(img.dtype)


class ToyAE(nn.Module):
    """4 x 8 x 8 compression, 3 pixel channels <-> 4 latent channels; causal (first frame alone) or not."""

    def __init__(self, causal: bool):
        super().__init__()
        self.scale = nn.Parameter(torch.tensor(0.5))
        self.causal = causal
        self.compression = (4, 8, 8)

    def encode(self, x):
        b, c, t, h, w = x.shape
        x = x.float().reshape(b, c, t, h // 8, 8, w // 8, 8).mean(dim=(4, 6))
        x = x[:, :, ::4] if self.causal else x[:, :, : t // 4 * 4].reshape(b, c, max(t // 4, 1), -1, h // 8, w // 8).mean(3) \
            if t >= 4 else x[:, :, :1]
        z = torch.cat((x, x.mean(1, keepdim=True)), dim=1) * self.scale.float()
        return z.to(self.scale.dtype)

    def decode(self, z):
        z = z.float()[:, :3] / self.scale.float() + 0.05 * z.float()[:, 3:]
        z = z.repeat_interleave(8, dim=3).repeat_interleave(8, dim=4)
        if self.causal:
            z = torch.cat((z[:, :, :1], z[:, :, 1:].repeat_interleave(4, dim=2)), dim=2)
        else:
            z = z.repeat_interleave(4, dim=2)
        return z.to(self.scale.dtype)


def _code(s: str) -> float:
    return (sum(ord(ch) * (i + 1) for i, ch in enumerate(s)) % 997) / 997.0


def toy_t5(prompts, added_tokens=0, seq_align=1):
    base = torch.tensor([_code(p) for p in prompts])[:, None, None]
    return base + 0.01 * torch.arange(6.0)[None, :, None] + 0.001 * torch.arange(8.0)[None, None, :] + 1e-4 * added_tokens * seq_align


def toy_clip(prompts):
    return torch.tensor([_code(p[::-1]) for p in prompts])[:, None] + 0.01 * torch.arange(8.0)[None, :]


def reference_media():
    """Pixel-space references [C, T, H, W] by 'path'."""
    g = torch.Generator().manual_seed(11)
    return {"img_a": torch.rand(3, 1, 32, 48, generator=g) * 2 - 1, "img_b": torch.rand(3, 1, 32, 48, generator=g) * 2 - 1,
            "clip_a": torch.rand(3, 40, 32, 48, generator=g) * 2 - 1}


# (name, option fields, api_fn keyword arguments) - every conditioning kind, both VAE kinds, both denoisers
SCENARIOS = [
    ("t2v_causal", dict(height=32, width=48, num_frames=17, num_steps=6, guidance=7.5, guidance_img=3.0, temporal_reduction=4,
                        is_causal_vae=True, seed=3), dict(cond_type="t2v", text=["a cat", "a dog"], neg=["blurry", "dark"])),
    ("i2v_head_causal_osci", dict(height=32, width=48, num_frames=17, num_steps=12, guidance=7.5, guidance_img=3.0, text_osci=True,
                                  image_osci=True, scale_temporal_osci=True, temporal_reduction=4, is_causal_vae=True, seed=4),
     dict(cond_type="i2v_head", text=["a cat"], ref=["img_a"])),
    ("i2v_loop_noncausal", dict(height=32, width=48, num_frames=16, num_steps=5, guidance=6.0, guidance_img=2.0, temporal_reduction=4,
                                is_causal_vae=False, seed=5, flow_shift=2.5), dict(cond_type="i2v_loop", text=["a fox"], ref=["img_a;img_b"])),
    ("i2v_tail_noncausal", dict(height=32, width=48, num_frames=16, num_steps=4, guidance=6.0, guidance_img=2.0, temporal_reduction=4,
                                is_causal_vae=False), dict(cond_type="i2v_tail", text=["a fox", "an owl"], ref=["img_b", ""], seed=9)),
    ("v2v_head_causal", dict(height=32, width=48, num_frames=65, num_steps=4, guidance=7.5, guidance_img=3.0, temporal_reduction=4,
                             is_causal_vae=True, seed=6, shift=False), dict(cond_type="v2v_head", text=["a bird"], ref=["clip_a"])),
    ("missing_ref_falls_back_to_t2v", dict(height=30, width=40, num_frames=5, num_steps=3, guidance=5.0, guidance_img=2.0,
                                           temporal_reduction=4, is_causal_vae=True, seed=7), dict(cond_type="i2v_head", text=["a cat"])),
    ("distilled_image", dict(height=32, width=48, num_frames=1, num_steps=4, guidance=3.5, method="distill", seed=8),
     dict(cond_type="t2v", text=["a tree", "a hill"])),
]


def toy_model(x, timestep, y, mask=None, x_mask=None, **kw):
    v = torch.tanh(0.8 * x.float() + y.float().mean(dim=(1, 2, 3))[:, None, None, None, None])
    v = v * (0.5 + timestep.float()[:, None, None, None, None] / 1000.0)
    return torch.cat((v, 0.1 * x.float()), dim=1)
