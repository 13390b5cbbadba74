"""The reference's rectified-flow sampler (`opensora/utils/sampling.py`) with the same names and argument meaning:
options (`SamplingOption` :28-79, `sanitize_sampling_option` :82-117), schedule (`time_shift` :295,
`get_res_lin_function` :299-304, `get_schedule` :307-332), noise / packing (`get_noise` :335-372, `pack` / `unpack`
:375-393), oscillating guidance (`get_oscillation_gs` :120-133), the denoisers (`I2VDenoiser` :158-245 - its per-step CFG
combine + Euler update runs as ONE osb200 kernel, `osb_cfg_euler`, instead of ~7 elementwise torch ops -
`DistilledDenoiser` :248-281), model-input assembly (`prepare` :401-459, `prepare_ids` :462-508) and the request ->
video closure `prepare_api` (:562-726) around denoiser + VAE.  Model construction from a config (`prepare_models`
:511-559: text encoders, LoRA, mmengine) stays with the caller (SURVEY.md 2 #14-15)."""
from __future__ import annotations

import math
import os
import random
from abc import ABC, abstractmethod
from dataclasses import dataclass, replace

import torch
from torch import Tensor

from opensora.datasets.aspect import get_image_size
from opensora.utils.inference import SamplingMethod, collect_references_batch, prepare_inference_condition


@dataclass
class SamplingOption:
    """sampling.py:28-79 (field names and defaults are the request format of the inference scripts)."""

    width: int | None = None
    height: int | None = None
    resolution: str | None = None        # with aspect_ratio: overrides height / width
    aspect_ratio: str | None = None
    num_frames: int = 1
    num_steps: int = 50
    guidance: float = 4.0                # classifier-free guidance, text
    text_osci: bool = False
    guidance_img: float | None = None    # classifier-free guidance, image / video condition
    image_osci: bool = False
    scale_temporal_osci: bool = False
    seed: int | None = None
    shift: bool = True
    method: str | SamplingMethod = SamplingMethod.I2V
    temporal_reduction: int = 1
    is_causal_vae: bool = False
    flow_shift: float | None = None


def sanitize_sampling_option(sampling_option: SamplingOption) -> SamplingOption:
    """Resolve (resolution, aspect_ratio) to a size, round height / width UP to multiples of 16, turn a method name into
    the enum (:82-117)."""
    opt = sampling_option
    if opt.resolution is not None or opt.aspect_ratio is not None:
        assert opt.resolution is not None and opt.aspect_ratio is not None, "Both resolution and aspect ratio must be provided"
        height, width = get_image_size(opt.resolution, opt.aspect_ratio, training=False)
    else:
        assert opt.height is not None and opt.width is not None, "Both height and width must be provided"
        height, width = opt.height, opt.width
    changes = dict(height=-(-height // 16) * 16, width=-(-width // 16) * 16)
    if isinstance(opt.method, str):
        changes["method"] = SamplingMethod(opt.method)
    return replace(opt, **changes)


def time_shift(alpha: float, t: Tensor) -> Tensor:
    return alpha * t / (1 + (alpha - 1) * t)


def get_res_lin_function(x1: float = 256, y1: float = 1, x2: float = 4096, y2: float = 3):
    m = (y2 - y1) / (x2 - x1)
    b = y1 - m * x1
    return lambda x: m * x + b


def get_schedule(num_steps: int, image_seq_len: int, num_frames: int, shift_alpha: float | None = None,
                 base_shift: float = 1, max_shift: float = 3, shift: bool = True) -> list[float]:
    timesteps = torch.linspace(1, 0, num_steps + 1)
    if shift:
        if shift_alpha is None:
            shift_alpha = get_res_lin_function(y1=base_shift, y2=max_shift)(image_seq_len)
            shift_alpha *= math.sqrt(num_frames)
        timesteps = time_shift(shift_alpha, timesteps)
    return timesteps.tolist()


def get_noise(num_samples: int, height: int, width: int, num_frames: int, device, dtype, seed: int, patch_size: int = 2,
              channel: int = 16) -> Tensor:
    D = int(os.environ.get("AE_SPATIAL_COMPRESSION", 16))
    return torch.randn(num_samples, channel, num_frames, patch_size * math.ceil(height / D), patch_size * math.ceil(width / D),
                       device=device, dtype=dtype, generator=torch.Generator(device=device).manual_seed(seed))


def pack(x: Tensor, patch_size: int = 2) -> Tensor:
    """"b c t (h ph) (w pw) -> b (t h w) (c ph pw)" (:375-378)."""
    b, c, t, hh, ww = x.shape
    h, w = hh // patch_size, ww // patch_size
    x = x.reshape(b, c, t, h, patch_size, w, patch_size).permute(0, 2, 3, 5, 1, 4, 6)
    return x.reshape(b, t * h * w, c * patch_size * patch_size)


def unpack(x: Tensor, height: int, width: int, num_frames: int, patch_size: int = 2) -> Tensor:
    """"b (t h w) (c ph pw) -> b c t (h ph) (w pw)" (:381-393)."""
    D = int(os.environ.get("AE_SPATIAL_COMPRESSION", 16))
    h, w, t = math.ceil(height / D), math.ceil(width / D), num_frames
    b, _, cpp = x.shape
    c = cpp // (patch_size * patch_size)
    x = x.reshape(b, t, h, w, c, patch_size, patch_size).permute(0, 4, 1, 2, 5, 3, 6)
    return x.reshape(b, c, t, h * patch_size, w * patch_size)


def get_oscillation_gs(guidance_scale: float, i: int, force_num=10):
    if i < force_num or (i >= force_num and i % 2 == 0):
        return guidance_scale
    return 1.0


class Denoiser(ABC):
    @abstractmethod
    def denoise(self, model, **kwargs) -> Tensor:
        """Run the sampling loop."""

    @abstractmethod
    def prepare_guidance(self, text: list[str], optional_models: dict, device, dtype, **kwargs):
        """Method-specific classifier-free-guidance inputs; may extend `text`.  Returns (text, extra model inputs)."""


class I2VDenoiser(Denoiser):
    """`I2VDenoiser.denoise` (:159-226): 3-way CFG batch (cond / uncond-text / uncond-text+image), Euler steps."""

    def prepare_guidance(self, text, optional_models, device, dtype, **kwargs):
        """:228-245.  The prompt list grows to [text, neg, neg] - the three CFG branches."""
        neg = kwargs.get("neg", None)
        if neg is None:
            neg = [""] * len(text)
        return text + neg + neg, {"guidance_img": kwargs.pop("guidance_img")}

    def denoise(self, model, **kwargs) -> Tensor:
        import osb200

        img = kwargs.pop("img")
        timesteps = kwargs.pop("timesteps")
        guidance = kwargs.pop("guidance")
        guidance_img = kwargs.pop("guidance_img")
        masks = kwargs.pop("masks")
        masked_ref = kwargs.pop("masked_ref")
        kwargs.pop("sigma_min")
        text_osci = kwargs.pop("text_osci", False)
        image_osci = kwargs.pop("image_osci", False)
        scale_temporal_osci = kwargs.pop("scale_temporal_osci", False)
        patch_size = kwargs.pop("patch_size", 2)

        guidance_vec = torch.full((img.shape[0],), guidance, device=img.device, dtype=img.dtype)
        b, c, t, w, h = masked_ref.size()  # (sic) the reference names them this way (:186)
        cond = pack(torch.cat((masks, masked_ref), dim=1), patch_size=patch_size)
        kwargs["cond"] = torch.cat([cond, cond, torch.zeros_like(cond)], dim=0)  # step-invariant: hoisted out of the loop
        x = img[: len(img) // 3].contiguous()
        for i, (t_curr, t_prev) in enumerate(zip(timesteps[:-1], timesteps[1:])):
            t_vec = torch.full((img.shape[0],), t_curr, dtype=img.dtype, device=img.device)
            pred = model(img=torch.cat([x, x, x], dim=0), **kwargs, timesteps=t_vec, guidance=guidance_vec)
            text_gs = get_oscillation_gs(guidance, i) if text_osci else guidance
            image_gs = get_oscillation_gs(guidance_img, i) if image_osci else guidance_img
            gmap = None
            if image_gs > 1.0 and scale_temporal_osci:
                upper = torch.linspace(image_gs, 1.0, len(timesteps))[i]
                g5 = torch.linspace(1.0, upper, t)[None, None, :, None, None].repeat(b, c, 1, h, w)
                gmap = pack(g5, patch_size=patch_size).to(pred.device, pred.dtype).contiguous()
                image_gs = 1.0
            pc, pu, pu2 = (p.contiguous() for p in pred.chunk(3, dim=0))
            # pred = uncond_2 + image_gs*(uncond - uncond_2) + text_gs*(cond - uncond); x += (t_prev - t_curr)*pred  (:219-222)
            x = osb200.cfg_euler(pc, pu, pu2, x, g_txt=float(text_gs), g_img=float(image_gs), g_img_map=gmap,
                                 dt=float(t_prev - t_curr))
        return x


class DistilledDenoiser(Denoiser):
    """:248-281: guidance-distilled model, one forward per step, plain Euler update (one axpy on a latent-sized tensor)."""

    def denoise(self, model, **kwargs) -> Tensor:
        img = kwargs.pop("img")
        timesteps = kwargs.pop("timesteps")
        guidance = kwargs.pop("guidance")
        guidance_vec = torch.full((img.shape[0],), guidance, device=img.device, dtype=img.dtype)
        for t_curr, t_prev in zip(timesteps[:-1], timesteps[1:]):
            t_vec = torch.full((img.shape[0],), t_curr, dtype=img.dtype, device=img.device)
            pred = model(img=img, **kwargs, timesteps=t_vec, guidance=guidance_vec)
            img = img + (t_prev - t_curr) * pred
        return img

    def prepare_guidance(self, text, optional_models, device, dtype, **kwargs):
        return text, {}


SamplingMethodDict = {SamplingMethod.I2V: I2VDenoiser(), SamplingMethod.DISTILLED: DistilledDenoiser()}


def _position_ids(bs: int, t: int, h: int, w: int) -> Tensor:
    """[bs, t*h*w, 3] = (frame, row, column) of every latent patch: the `ids` the 3-axis RoPE is built from."""
    grid = torch.stack(torch.meshgrid(torch.arange(t), torch.arange(h), torch.arange(w), indexing="ij"), dim=-1)
    return grid.reshape(1, t * h * w, 3).float().repeat(bs, 1, 1)


def _broadcast_batch(x: Tensor, bs: int) -> Tensor:
    return x.repeat(bs, *([1] * (x.dim() - 1))) if x.shape[0] == 1 and bs > 1 else x


def prepare(t5, clip, img: Tensor, prompt: str | list[str], seq_align: int = 1, patch_size: int = 2) -> dict[str, Tensor]:
    """:401-459.  Latent noise [b, c, t, H, W] + prompts -> the denoiser's inputs: packed `img`, `img_ids` (positions for
    RoPE), `txt` (T5 tokens; the encoder is told how many image tokens follow so it can align the joint length), zero
    `txt_ids`, `y_vec` (CLIP pooled)."""
    _, c, t, h, w = img.shape
    device, dtype = img.device, img.dtype
    prompt = [prompt] if isinstance(prompt, str) else prompt
    bs = len(prompt)
    tokens = pack(img, patch_size=patch_size)
    if tokens.shape[0] != bs:
        tokens = tokens.repeat(bs // tokens.shape[0], 1, 1)
    img_ids = _position_ids(bs, t, h // patch_size, w // patch_size)
    txt = _broadcast_batch(t5(prompt, added_tokens=img_ids.shape[1], seq_align=seq_align), bs)
    vec = _broadcast_batch(clip(prompt), bs)
    return {"img": tokens, "img_ids": img_ids.to(device, dtype), "txt": txt.to(device, dtype),
            "txt_ids": torch.zeros(bs, txt.shape[1], 3).to(device, dtype), "y_vec": vec.to(device, dtype)}


def prepare_ids(img: Tensor, t5_embedding: Tensor, clip_embedding: Tensor) -> dict[str, Tensor]:
    """:462-508: `prepare` with pre-computed text embeddings (the training / cached-embedding path; patch size 2)."""
    bs, _, t, h, w = img.shape
    device, dtype = img.device, img.dtype
    txt = _broadcast_batch(t5_embedding, bs)
    return {"img": pack(img, patch_size=2), "img_ids": _position_ids(bs, t, h // 2, w // 2).to(device, dtype),
            "txt": txt.to(device, dtype), "txt_ids": torch.zeros(bs, txt.shape[1], 3).to(device, dtype),
            "y_vec": _broadcast_batch(clip_embedding, bs).to(device, dtype)}


def prepare_models(cfg, device, dtype, offload_model: bool = False):
    """:511-559.  Builds (model, model_ae, model_t5, model_clip, optional_models) from the config's `model`, `ae`, `t5` and
    `clip` dicts through the registry, with `device_map` / `torch_dtype` as the reference passes them;
    `pretrained_lora_path` goes through `load_lora`.  The text-to-image-to-video models (`img_flux`, `img_flux_ae`) need
    the Flux image autoencoder, which is not registered here."""
    from opensora.registry import MODELS, build_module

    if cfg.get("img_flux", None) is not None and "autoencoder_2d" not in MODELS:
        raise KeyError("img_flux_ae needs the Flux image autoencoder (type 'autoencoder_2d'), which is not registered in "
                       "this package")
    model_device = "cpu" if offload_model and cfg.get("img_flux", None) is not None else device
    model = build_module(cfg.get("model"), MODELS, device_map=model_device, torch_dtype=dtype).eval()
    model_ae = build_module(cfg.get("ae"), MODELS, device_map=model_device, torch_dtype=dtype).eval()
    model_t5 = build_module(cfg.get("t5"), MODELS, device_map=device, torch_dtype=dtype).eval()
    model_clip = build_module(cfg.get("clip"), MODELS, device_map=device, torch_dtype=dtype).eval()
    if cfg.get("pretrained_lora_path", None) is not None:
        from opensora.utils.lora import load_lora

        model = load_lora(model, cfg.get("pretrained_lora_path"))
    optional_models = {}
    if cfg.get("img_flux", None) is not None:
        optional_models["img_flux"] = build_module(cfg.get("img_flux"), MODELS, device_map=device, torch_dtype=dtype).eval()
        optional_models["img_flux_ae"] = build_module(cfg.get("img_flux_ae"), MODELS, device_map=device,
                                                      torch_dtype=dtype).eval()
    return model, model_ae, model_t5, model_clip, optional_models


def prepare_api(model, model_ae, model_t5, model_clip, optional_models: dict):
    """:562-726.  Returns `api_fn(opt, cond_type="t2v", seed=None, sigma_min=1e-5, text=None, neg=None, patch_size=2,
    channel=16, **kwargs)`: noise -> schedule -> guidance prompts -> model inputs -> conditioning -> denoise -> unpack ->
    re-insert the reference frames -> VAE decode -> crop to the requested frame count.  `ref=` entries are ';'-separated media
    per prompt (see `opensora.utils.inference.collect_references_batch`; `reader=` plugs in a file decoder)."""

    @torch.inference_mode()
    def api_fn(opt: SamplingOption, cond_type: str = "t2v", seed: int = None, sigma_min: float = 1e-5, text: list[str] = None,
               neg: list[str] = None, patch_size: int = 2, channel: int = 16, **kwargs):
        p = next(model.parameters())
        device, dtype = p.device, p.dtype
        if seed is None:   # an explicit seed wins over the option's; neither -> random
            seed = opt.seed if opt.seed is not None else random.randint(0, 2**32 - 1)
        if opt.num_frames == 1:
            num_frames = 1
        elif opt.is_causal_vae:
            num_frames = (opt.num_frames - 1) // opt.temporal_reduction + 1
        else:
            num_frames = opt.num_frames // opt.temporal_reduction
        z = get_noise(len(text), opt.height, opt.width, num_frames, device, dtype, seed, patch_size=patch_size,
                      channel=channel // (patch_size**2))
        denoiser = SamplingMethodDict[opt.method]

        references = [None] * len(text)
        if cond_type != "t2v" and "ref" in kwargs:
            references = collect_references_batch(kwargs.pop("ref"), cond_type, model_ae, (opt.height, opt.width),
                                                  is_causal=opt.is_causal_vae, reader=kwargs.pop("reader", None))
        elif cond_type != "t2v":
            print("your csv file doesn't have a ref column or is not processed properly. will default to cond_type t2v!")
            cond_type = "t2v"

        timesteps = get_schedule(opt.num_steps, (z.shape[-1] * z.shape[-2]) // patch_size**2, num_frames, shift=opt.shift,
                                 shift_alpha=opt.flow_shift)
        text, extra = denoiser.prepare_guidance(text=text, optional_models=optional_models, device=device, dtype=dtype, neg=neg,
                                                guidance_img=opt.guidance_img)
        inp = prepare(model_t5, model_clip, z, prompt=text, patch_size=patch_size)
        inp.update(extra)
        if opt.method in (SamplingMethod.I2V,):
            inp["masks"], inp["masked_ref"] = prepare_inference_condition(z, cond_type, ref_list=references, causal=opt.is_causal_vae)
            inp["sigma_min"] = sigma_min

        x = denoiser.denoise(model, **inp, timesteps=timesteps, guidance=opt.guidance, text_osci=opt.text_osci,
                             image_osci=opt.image_osci,
                             scale_temporal_osci=(opt.scale_temporal_osci and "i2v" in cond_type),   # not for v2v / t2v
                             flow_shift=opt.flow_shift, patch_size=patch_size)
        x = unpack(x, opt.height, opt.width, num_frames, patch_size=patch_size)

        # the conditioned latent frames are the reference latents themselves (first prompt of the batch only, as upstream)
        pinned = {"i2v_head": ((0, 0),), "i2v_tail": ((-1, 0),), "i2v_loop": ((0, 0), (-1, 1))}.get(cond_type, ())
        for frame, which in pinned:
            x[0, :, frame] = references[0][which][:, 0]

        x = model_ae.decode(x)
        x = x[:, :, : opt.num_frames]
        if not opt.is_causal_vae and pinned:
            # a non-causal AE turns each pinned latent frame into `compression[0]` identical pixel frames: keep one
            dup = model_ae.compression[0] - 1
            first = dup if cond_type in ("i2v_head", "i2v_loop") else 0
            last = x.shape[2] - (dup if cond_type in ("i2v_tail", "i2v_loop") else 0)
            x = x[:, :, first:last]
        return x

    return api_fn
