"""`AutoencoderKLCausal3D` / `CausalVAE3D_HUNYUAN` with the reference's public surface
(`opensora/models/hunyuan_vae/autoencoder_kl_causal_3d.py:59-146,269-358,554-638`): registry key
`"hunyuan_vae"`, `encode / decode / forward / get_latent_size`, `scale_factor`, `shift_factor`, `z_channels`,
compression ratios, tiling toggles, identical state-dict keys — arithmetic on libosb200 (sm_90a).

Untiled (`:298-304`, `:318-335`) is the fast path wherever the activations fit (it avoids the ~1.65x tile-overlap
recompute); on one 80 GB H100 that holds for 720p videos of about 33 frames, longer ones need tiling.  The reference's tiled / blended modes (`:384-552`) are reproduced with the
same tile grid, overlap, in-place blending order and cropping, because their numerics differ from untiled by
construction (per-tile GroupNorm statistics and causal start) and a caller that enables tiling must get the
reference's result; every tile runs through the same osb200 encoder / decoder."""
from __future__ import annotations

from dataclasses import dataclass

import torch
import torch.nn as nn

from opensora.registry import MODELS
from opensora.utils.lora import refuse_adapters

from .vae import DecoderCausal3D, DiagonalGaussianDistribution, EncoderCausal3D


@dataclass
class AutoEncoder3DConfig:
    from_pretrained: str | None = None
    act_fn: str = "silu"
    in_channels: int = 3
    out_channels: int = 3
    latent_channels: int = 16
    layers_per_block: int = 2
    norm_num_groups: int = 32
    scale_factor: float = 0.476986
    shift_factor: float = 0
    time_compression_ratio: int = 4
    spatial_compression_ratio: int = 8
    mid_block_add_attention: bool = True
    block_out_channels: tuple = (128, 256, 512, 512)
    sample_size: int = 256
    sample_tsize: int = 64
    use_slicing: bool = False
    use_spatial_tiling: bool = False
    use_temporal_tiling: bool = False
    tile_overlap_factor: float = 0.25
    dropout: float = 0.0
    channel: bool = False


class AutoencoderKLCausal3D(nn.Module):
    def __init__(self, config: AutoEncoder3DConfig):
        super().__init__()
        self.config = config
        self.scale_factor, self.shift_factor = config.scale_factor, config.shift_factor
        self.time_compression_ratio = config.time_compression_ratio
        self.spatial_compression_ratio = config.spatial_compression_ratio
        self.z_channels = config.latent_channels
        common = dict(block_out_channels=config.block_out_channels, layers_per_block=config.layers_per_block,
                      act_fn=config.act_fn, norm_num_groups=config.norm_num_groups,
                      time_compression_ratio=config.time_compression_ratio,
                      spatial_compression_ratio=config.spatial_compression_ratio,
                      mid_block_add_attention=config.mid_block_add_attention, dropout=config.dropout)
        self.encoder = EncoderCausal3D(in_channels=config.in_channels, out_channels=config.latent_channels, double_z=True, **common)
        self.decoder = DecoderCausal3D(in_channels=config.latent_channels, out_channels=config.out_channels, **common)
        self.quant_conv = nn.Conv3d(2 * config.latent_channels, 2 * config.latent_channels, kernel_size=1)
        self.post_quant_conv = nn.Conv3d(config.latent_channels, config.latent_channels, kernel_size=1)
        self.use_slicing = config.use_slicing
        self.use_spatial_tiling = config.use_spatial_tiling
        self.use_temporal_tiling = config.use_temporal_tiling
        self.tile_sample_min_tsize = config.sample_tsize
        self.tile_latent_min_tsize = config.sample_tsize // config.time_compression_ratio
        ss = config.sample_size[0] if isinstance(config.sample_size, (list, tuple)) else config.sample_size
        self.tile_sample_min_size = config.sample_size
        self.tile_latent_min_size = int(ss / (2 ** (len(config.block_out_channels) - 1)))
        self.tile_overlap_factor = config.tile_overlap_factor

    # ---- toggles (same names as the reference :148-189) ------------------------------------------------
    def enable_temporal_tiling(self, use_tiling: bool = True):
        self.use_temporal_tiling = use_tiling

    def disable_temporal_tiling(self):
        self.enable_temporal_tiling(False)

    def enable_spatial_tiling(self, use_tiling: bool = True):
        self.use_spatial_tiling = use_tiling

    def disable_spatial_tiling(self):
        self.enable_spatial_tiling(False)

    def enable_tiling(self, use_tiling: bool = True):
        self.enable_spatial_tiling(use_tiling)
        self.enable_temporal_tiling(use_tiling)

    def disable_tiling(self):
        self.enable_tiling(False)

    def enable_slicing(self):
        self.use_slicing = True

    def disable_slicing(self):
        self.use_slicing = False

    def enable_temporal_parallel(self, process_group=None):
        """Shard the VAE by frames over `process_group` (one process per GPU; None switches it off).  Every rank passes the
        SAME tensor to `encode` / `decode` and gets the whole result back; in between each rank works on its run of frames
        in every layer: convolutions take a one- or two-frame causal halo from the left neighbour, GroupNorm statistics are
        combined over the group, the mid block's frame-causal attention runs local queries against gathered keys / values
        (unet_causal_3d_blocks._TemporalShard), and one gather at the end rebuilds the result.  No reference counterpart
        (single-GPU VAE, tiled when short of memory; its channel-tensor-parallel policy is not reproduced); composes with
        spatial tiling, and inputs too short to shard (fewer than 2 latent frames per rank) run replicated."""
        import torch.distributed as dist

        if process_group is not None and dist.get_world_size(process_group) == 1:
            process_group = None
        self.decoder.shard_group = process_group
        self.encoder.shard_group = process_group

    def _mid_attentions(self):
        return [a for part in (self.encoder, self.decoder) for a in part.mid_block.attentions if a is not None]

    def enable_native_attention(self):
        """Run the mid block's frame-causal attention (encoder and decoder, untiled, tiled and frame-sharded) as ONE
        `osb_attn_frames` launch instead of one torch SDPA call per latent frame.  The kernel is built for one head of
        512 channels - the width of every released checkpoint's mid block; any other width is refused here, never run
        on another path.  Off by default: the default path still calls SDPA."""
        for a in self._mid_attentions():
            width = a.to_q.in_features
            if width != 512:
                raise ValueError(f"enable_native_attention: osb_attn_frames is built for a 512-wide mid block, this "
                                 f"model's is {width} wide (block_out_channels[-1])")
        for a in self._mid_attentions():
            a.native = True

    def disable_native_attention(self):
        for a in self._mid_attentions():
            a.native = False

    # ---- helpers -------------------------------------------------------------------------------------
    def _check(self):
        import osb200

        w = self.quant_conv.weight
        osb200.require_cuda_bf16(w, "AutoencoderKLCausal3D")
        return osb200

    @staticmethod
    def _to_ndhwc(x, cpad=None):
        x = x.permute(0, 2, 3, 4, 1)
        if cpad is not None and x.shape[-1] < cpad:
            x = torch.nn.functional.pad(x, (0, cpad - x.shape[-1]))
        return x.contiguous()

    @staticmethod
    def _to_ncdhw(x):
        return x.permute(0, 4, 1, 2, 3).contiguous()

    @staticmethod
    def _pointwise(osb, x2d, conv):
        """1x1x1 Conv3d == GEMM over channels-last rows.  osb_gemm_bf16 wants K, N multiples of 8: narrower (test-sized)
        latent widths are zero-padded on both sides; the production widths (16 / 32) take the direct path."""
        C = conv.weight.shape[0]
        w, b = conv.weight.reshape(C, C), conv.bias
        if C % 8 == 0:
            return osb.gemm(x2d, w, b)
        Cp = (C + 7) // 8 * 8
        wp = torch.zeros(Cp, Cp, dtype=w.dtype, device=w.device)
        wp[:C, :C] = w
        bp = torch.zeros(Cp, dtype=b.dtype, device=b.device)
        bp[:C] = b
        xp = torch.nn.functional.pad(x2d, (0, Cp - C))
        return osb.gemm(xp, wp, bp)[:, :C].contiguous()

    # ---- tile-level building blocks (NCDHW in / out, bf16) ----------------------------------------------------
    def _encode_moments(self, x):
        """encoder + quant_conv on one (tile of a) video -> moments [B, 2*latent, T', h, w]."""
        osb = self._check()
        h = self.encoder(self._to_ndhwc(x, cpad=8))
        nb, T, H, W, C2 = h.shape
        m = self._pointwise(osb, h.reshape(-1, C2), self.quant_conv)
        return self._to_ncdhw(m.view(nb, T, H, W, C2))

    def _decode_tile(self, z):
        """post_quant_conv + decoder on one (tile of a) latent."""
        osb = self._check()
        zl = self._to_ndhwc(z)
        nb, T, H, W, C = zl.shape
        zl = self._pointwise(osb, zl.reshape(-1, C), self.post_quant_conv)
        return self._to_ncdhw(self.decoder(zl.view(nb, T, H, W, C)))

    @staticmethod
    def _blend(a, b, extent, dim):
        """blend_v / blend_h / blend_t (:360-382): linear cross-fade of the first `extent` slices of `b` (in place) with
        the last `extent` slices of `a` along `dim`; one vectorised lerp instead of a Python loop per slice."""
        extent = min(a.shape[dim], b.shape[dim], extent)
        if extent <= 0:
            return b
        w = (torch.arange(extent, device=b.device, dtype=torch.float32) / extent).view([-1 if d == dim % 5 else 1 for d in range(5)])
        bs = b.narrow(dim, 0, extent)
        bs.copy_(a.narrow(dim, a.shape[dim] - extent, extent).float() * (1 - w) + bs.float() * w)
        return b

    def spatial_tiled_encode(self, x, return_moments: bool = False):
        """:384-434."""
        overlap = int(self.tile_sample_min_size * (1 - self.tile_overlap_factor))
        blend = int(self.tile_latent_min_size * self.tile_overlap_factor)
        limit = self.tile_latent_min_size - blend
        ts = self.tile_sample_min_size
        rows = [[self._encode_moments(x[:, :, :, i:i + ts, j:j + ts]) for j in range(0, x.shape[-1], overlap)]
                for i in range(0, x.shape[-2], overlap)]
        moments = self._stitch(rows, blend, limit)
        return moments if return_moments else DiagonalGaussianDistribution(moments)

    def spatial_tiled_decode(self, z):
        """:436-484."""
        overlap = int(self.tile_latent_min_size * (1 - self.tile_overlap_factor))
        blend = int(self.tile_sample_min_size * self.tile_overlap_factor)
        limit = self.tile_sample_min_size - blend
        tl = self.tile_latent_min_size
        rows = [[self._decode_tile(z[:, :, :, i:i + tl, j:j + tl]) for j in range(0, z.shape[-1], overlap)]
                for i in range(0, z.shape[-2], overlap)]
        return self._stitch(rows, blend, limit)

    def _stitch(self, rows, blend, limit):
        out_rows = []
        for i, row in enumerate(rows):
            out = []
            for j, tile in enumerate(row):
                if i > 0:
                    tile = self._blend(rows[i - 1][j], tile, blend, -2)
                if j > 0:
                    tile = self._blend(row[j - 1], tile, blend, -1)
                out.append(tile[:, :, :, :limit, :limit])
            out_rows.append(torch.cat(out, dim=-1))
        return torch.cat(out_rows, dim=-2)

    def temporal_tiled_encode(self, x):
        """:486-515."""
        overlap = int(self.tile_sample_min_tsize * (1 - self.tile_overlap_factor))
        blend = int(self.tile_latent_min_tsize * self.tile_overlap_factor)
        t_limit = self.tile_latent_min_tsize - blend
        row = []
        for i in range(0, x.shape[2], overlap):
            tile = x[:, :, i:i + self.tile_sample_min_tsize + 1]
            if self.use_spatial_tiling and (tile.shape[-1] > self.tile_sample_min_size or tile.shape[-2] > self.tile_sample_min_size):
                tile = self.spatial_tiled_encode(tile, return_moments=True)
            else:
                tile = self._encode_moments(tile)
            row.append(tile[:, :, 1:] if i > 0 else tile)
        return DiagonalGaussianDistribution(self._stitch_t(row, blend, t_limit))

    def temporal_tiled_decode(self, z):
        """:517-548."""
        overlap = int(self.tile_latent_min_tsize * (1 - self.tile_overlap_factor))
        blend = int(self.tile_sample_min_tsize * self.tile_overlap_factor)
        t_limit = self.tile_sample_min_tsize - blend
        row = []
        for i in range(0, z.shape[2], overlap):
            tile = z[:, :, i:i + self.tile_latent_min_tsize + 1]
            if self.use_spatial_tiling and (tile.shape[-1] > self.tile_latent_min_size or tile.shape[-2] > self.tile_latent_min_size):
                dec = self.spatial_tiled_decode(tile)
            else:
                dec = self._decode_tile(tile)
            row.append(dec[:, :, 1:] if i > 0 else dec)
        return self._stitch_t(row, blend, t_limit)

    def _stitch_t(self, row, blend, t_limit):
        out = []
        for i, tile in enumerate(row):
            if i > 0:
                tile = self._blend(row[i - 1], tile, blend, 2)
                out.append(tile[:, :, :t_limit])
            else:
                out.append(tile[:, :, :t_limit + 1])
        return torch.cat(out, dim=2)

    # ---- public API (:269-358, :554-622) -------------------------------------------------------------------
    def encode(self, x, sample_posterior=True, return_posterior=False, generator=None):
        self._check()
        refuse_adapters(self, "AutoencoderKLCausal3D")   # no LoRA path: never silently run the base model
        assert x.dim() == 5, "The input tensor should have 5 dimensions."
        x = x.to(self.quant_conv.weight.device, torch.bfloat16)
        if self.use_temporal_tiling and x.shape[2] > self.tile_sample_min_tsize:
            posterior = self.temporal_tiled_encode(x)
        elif self.use_spatial_tiling and (x.shape[-1] > self.tile_sample_min_size or x.shape[-2] > self.tile_sample_min_size):
            posterior = self.spatial_tiled_encode(x)
        else:
            posterior = DiagonalGaussianDistribution(self._encode_moments(x))
        z = posterior.sample(generator=generator) if sample_posterior else posterior.mode()
        z = self.scale_factor * (z - self.shift_factor)
        return (z, posterior) if return_posterior else z

    def _decode(self, z):
        if self.use_temporal_tiling and z.shape[2] > self.tile_latent_min_tsize:
            return self.temporal_tiled_decode(z)
        if self.use_spatial_tiling and (z.shape[-1] > self.tile_latent_min_size or z.shape[-2] > self.tile_latent_min_size):
            return self.spatial_tiled_decode(z)
        return self._decode_tile(z)

    def decode(self, z):
        self._check()
        refuse_adapters(self, "AutoencoderKLCausal3D")   # no LoRA path: never silently run the base model
        z = z.to(self.quant_conv.weight.device, torch.bfloat16) / self.scale_factor + self.shift_factor
        if self.use_slicing and z.shape[0] > 1:
            return torch.cat([self._decode(zs) for zs in z.split(1)])
        return self._decode(z)

    def forward(self, x, sample_posterior=True, generator=None):
        z, posterior = self.encode(x, return_posterior=True, sample_posterior=sample_posterior, generator=generator)
        return self.decode(z), posterior, z

    def get_last_layer(self):
        return self.decoder.conv_out.conv.weight

    def get_latent_size(self, input_size: list[int]) -> list[int]:
        """autoencoder_kl_causal_3d.py:615-622."""
        latent_size = [(input_size[0] - 1) // self.time_compression_ratio + 1]
        for i in range(1, 3):
            latent_size.append((input_size[i] - 1) // self.spatial_compression_ratio + 1)
        return latent_size


@MODELS.register_module("hunyuan_vae")
def CausalVAE3D_HUNYUAN(from_pretrained: str = None, device_map: str | torch.device = "cuda",
                        torch_dtype: torch.dtype = torch.bfloat16, **kwargs) -> AutoencoderKLCausal3D:
    """Same factory signature as autoencoder_kl_causal_3d.py:625-638."""
    fields = AutoEncoder3DConfig.__dataclass_fields__
    config = AutoEncoder3DConfig(from_pretrained=from_pretrained, **{k: v for k, v in kwargs.items() if k in fields})
    model = AutoencoderKLCausal3D(config)
    if from_pretrained:
        from opensora.utils.ckpt import load_checkpoint

        model = load_checkpoint(model, from_pretrained, device_map="cpu", strict=True)
    return model.to(device=device_map, dtype=torch_dtype) if torch.cuda.is_available() or str(device_map) == "cpu" \
        else model.to(dtype=torch_dtype)
