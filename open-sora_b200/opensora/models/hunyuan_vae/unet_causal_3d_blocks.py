"""Causal 3D VAE building blocks on the osb200 kernels (channels-last NDHWC inside, bf16).

Same class names, constructor meaning and state-dict keys as the reference's
`opensora/models/hunyuan_vae/unet_causal_3d_blocks.py` (`CausalConv3d` :63-96, `UpsampleCausal3D` :98-158,
`DownsampleCausal3D` :160-181, `ResnetBlockCausal3D` :184-259, `UNetMidBlockCausal3D` :262-355,
`DownEncoderBlockCausal3D`, `UpDecoderBlockCausal3D`).  The nn.Modules hold parameters only; `forward` takes and
returns **NDHWC bf16** tensors and runs on libosb200: GroupNorm statistics (`osb_group_stats`), one fused
GN-apply + SiLU + nearest-upsample + replicate-pad pass (`osb_vae_prep`) and the implicit-GEMM convolution
(`osb_conv3d_ndhwc`, wgmma, residual add fused in the epilogue).  1x1x1 convolutions are plain GEMMs.
No CPU / eager fallback."""
from __future__ import annotations

import torch
import torch.nn as nn


def _osb():
    import osb200

    return osb200


class _TemporalShard:
    """Frame-sharded decode (SURVEY.md 8e "VAE T-shard with halo").  While `group` is set, every rank of it holds a contiguous
    run of frames of the same video (rank order = frame order) and each 3x3x3 `CausalConv3d`
      * normalises with GroupNorm statistics over ALL ranks' frames (per-rank mean / variance combined with their element
        counts - the parallel-variance identity, so no second pass over the activations), and
      * takes the two causal context frames it needs from its left neighbour (one point-to-point message per convolution)
        instead of the replicate padding, which only rank 0 - the owner of the first frame - applies;
    and the mid block's frame-causal attention keeps its queries local and gathers keys / values (`_gather_frames`).
    The reference has no counterpart (its VAE runs on one GPU, tiled when memory is short: autoencoder_kl_causal_3d.py:
    454-560); results equal the un-sharded decode up to the rounding of the combined statistics.

    `start` is the global index of this rank's first frame at the current layer.  Only the encoder needs it: a
    temporally strided convolution reads windows that begin at even (padded) positions, so how many context frames a rank
    needs from its left neighbour - 2 or 1 - depends on the parity of its first frame; the convolution updates it."""

    group = None
    start = None


class temporal_shard:
    """`with temporal_shard(group): ...` - scope in which CausalConv3d treats its input as this rank's frame run."""

    def __init__(self, group, start: int | None = None):
        self.group, self.start = group, start

    def __enter__(self):
        self.prev = (_TemporalShard.group, _TemporalShard.start)
        _TemporalShard.group, _TemporalShard.start = self.group, self.start
        return self

    def __exit__(self, *exc):
        _TemporalShard.group, _TemporalShard.start = self.prev
        return False


def frame_partition(frames: int, parts: int) -> list[int]:
    """Contiguous split of `frames` over `parts` ranks, the remainder on the lowest ranks (rank 0 owns the first frame, whose
    upsampling rule differs)."""
    base, rem = divmod(frames, parts)
    return [base + (1 if r < rem else 0) for r in range(parts)]


def _combine_group_stats(stats, count: int, eps: float, group):
    """(mean, rstd) fp32 [nb, G, 2] of this rank's `count` elements per group -> the statistics of the union over the group's
    ranks: mean = sum n_r m_r / N,  var = sum n_r (v_r + (m_r - mean)^2) / N  (no cancellation, so fp32 is enough)."""
    import torch.distributed as dist

    P = dist.get_world_size(group)
    mean, rstd = stats[..., 0], stats[..., 1]
    var = (1.0 / (rstd * rstd) - eps).clamp_min(0.0)
    mine = torch.stack((mean, var, torch.full_like(mean, float(count))), dim=-1).contiguous()
    flat = torch.empty((P * mine.shape[0],) + tuple(mine.shape[1:]), dtype=mine.dtype, device=mine.device)
    dist.all_gather_into_tensor(flat, mine, group=group)   # rank-major concatenation along dim 0
    every = flat.view((P,) + tuple(mine.shape))
    m, v, n = every[..., 0].double(), every[..., 1].double(), every[..., 2].double()
    total = n.sum(0)
    gmean = (n * m).sum(0) / total
    gvar = (n * (v + (m - gmean) ** 2)).sum(0) / total
    return torch.stack((gmean, torch.rsqrt(gvar + eps)), dim=-1).float().contiguous()


def _left_halo(x, frames: int, group, send_frames: int | None = None):
    """Send my last `send_frames` (default `frames`) frames to the right neighbour, return the left neighbour's last
    `frames` (None on rank 0)."""
    import torch.distributed as dist

    P, r = dist.get_world_size(group), dist.get_rank(group)
    send_frames = frames if send_frames is None else send_frames
    if x.shape[1] < max(frames, send_frames):
        raise ValueError(f"temporal shard: {x.shape[1]} local frame(s), the causal halo needs {max(frames, send_frames)}")
    ops, halo = [], None
    if r + 1 < P:
        tail = x[:, -send_frames:].contiguous()
        ops.append(dist.P2POp(dist.isend, tail, dist.get_global_rank(group, r + 1), group))
    if r > 0:
        halo = torch.empty((x.shape[0], frames) + tuple(x.shape[2:]), dtype=x.dtype, device=x.device)
        ops.append(dist.P2POp(dist.irecv, halo, dist.get_global_rank(group, r - 1), group))
    for w in dist.batch_isend_irecv(ops) if ops else ():
        w.wait()
    return halo


class CausalConv3d(nn.Module):
    """Parameter container + launcher.  `forward(x, norm=..., silu=..., up=..., residual=...)`: the optional
    GroupNorm(+SiLU) and nearest upsample that PRECEDE this convolution in the reference are folded into the
    padding pass that builds its input."""

    def __init__(self, chan_in, chan_out, kernel_size=3, stride=1, dilation=1, pad_mode="replicate", **kwargs):
        super().__init__()
        assert pad_mode == "replicate" and dilation == 1
        self.kernel_size = kernel_size
        self.stride = (stride,) * 3 if isinstance(stride, int) else tuple(stride)
        self.time_causal_padding = (kernel_size // 2,) * 4 + (kernel_size - 1, 0)
        self.conv = nn.Conv3d(chan_in, chan_out, kernel_size, stride=self.stride, **kwargs)  # parameters only
        self._packed = None

    def _apply(self, fn, *a, **k):
        self._packed = None
        return super()._apply(fn, *a, **k)

    def _weights(self):
        if self._packed is None:
            osb = _osb()
            w, b = self.conv.weight, self.conv.bias
            cout, cin = w.shape[:2]
            co = (cout + 7) // 8 * 8
            if self.kernel_size == 1:
                wp = torch.zeros(co, cin, dtype=torch.bfloat16, device=w.device)
                wp[:cout] = w.reshape(cout, cin)
                narrow, cp = False, cin
            else:
                narrow = cin <= 16
                cp = ((cin + 7) // 8 * 8 if cin <= 8 else 16) if narrow else (cin + 63) // 64 * 64
                wp = osb.pack_conv_weight(w.detach(), cp, narrow, cout_pad=co)
            bp = None
            if b is not None:
                bp = torch.zeros(co, dtype=torch.bfloat16, device=w.device)
                bp[:cout] = b.detach()
            self._packed = (wp.contiguous(), bp, narrow, cp, cout)
        return self._packed

    def forward(self, x, norm: nn.GroupNorm | None = None, silu: bool = False, up=(1, 1, 1), residual=None):
        osb = _osb()
        osb.require_cuda_bf16(x, "hunyuan_vae CausalConv3d (channels-last inside)")
        wp, bp, narrow, cp, cout = self._weights()
        if x.shape[-1] % 8:  # e.g. a 4-channel latent: zero-pad channels once (weights are zero there too)
            x = torch.nn.functional.pad(x, (0, -x.shape[-1] % 8))
        nb, T, H, W, C = x.shape
        if self.kernel_size == 1:
            assert norm is None and not silu and up == (1, 1, 1)
            y = osb.gemm(x.reshape(-1, C), wp, bp, epilogue=osb.EPI_BIAS if residual is None else osb.EPI_BIAS_GATE_RES,
                         residual=None if residual is None else residual.reshape(-1, wp.shape[0]))
            return y.view(nb, T, H, W, wp.shape[0])
        stats = gamma = beta = None
        groups = 1
        shard = _TemporalShard.group
        if norm is not None:
            groups = norm.num_groups
            stats = osb.group_stats(x, groups, norm.eps)
            gamma, beta = norm.weight, norm.bias
            if shard is not None:
                stats = _combine_group_stats(stats, T * H * W * (C // groups), norm.eps, shard)
        pad_t = self.kernel_size - 1
        if shard is not None:
            # Causal context across the shard boundary.
            #  * stride 1, no temporal upsample: the two frames in front of my first one = the left neighbour's last two.
            #  * x2 temporal upsample (decoder): both are copies of its last frame (also when that frame is the video's first,
            #    whose single copy the replicate padding doubles): the halo frame lands on `osb_vae_prep`'s first-frame rule
            #    (one copy) and ONE replicate-padded frame supplies the second.
            #  * temporal stride 2 (encoder): output j reads frames 2j-2 .. 2j; my first output is j0 = ceil(start / 2), so I
            #    need start - (2 j0 - 2) = 2 (even start) or 1 (odd start) frames of context, and my right neighbour - whose
            #    first frame is start + T - needs the same rule applied to its own parity.
            assert self.kernel_size == 3 and self.stride[0] in (1, 2), "temporal shard: 3x3x3 convolutions, temporal stride 1 or 2"
            if self.stride[0] == 2:
                assert up[0] == 1 and _TemporalShard.start is not None, "temporal shard: strided convolution needs the frame offset"
                start = _TemporalShard.start
                need, give = 2 - start % 2, 2 - (start + T) % 2
                halo = _left_halo(x, need, shard, send_frames=give)
                _TemporalShard.start = (start + 1) // 2
            else:
                halo = _left_halo(x, 2 if up[0] == 1 else 1, shard)
            if halo is not None:
                x = torch.cat((halo, x), dim=1)
                pad_t = 0 if up[0] == 1 else 1
        xp = osb.vae_prep(x, stats=stats, gamma=gamma, beta=beta, groups=groups, silu=silu, up=up,
                          pad=(pad_t, self.kernel_size // 2, self.kernel_size // 2), cp=cp)
        tp, hp, wpd = xp.shape[1:4]
        st, sh, sw = self.stride
        k = self.kernel_size
        out_thw = ((tp - k) // st + 1, (hp - k) // sh + 1, (wpd - k) // sw + 1)
        y = osb.conv3d(xp, wp, bp, out_thw=out_thw, stride=self.stride, taps=(k, k, k), narrow=narrow, residual=residual)
        return y if wp.shape[0] == cout else y[..., :cout]


class UpsampleCausal3D(nn.Module):
    def __init__(self, channels, out_channels=None, kernel_size=3, bias=True, upsample_factor=(2, 2, 2)):
        super().__init__()
        self.channels, self.out_channels = channels, out_channels or channels
        self.upsample_factor = tuple(upsample_factor)
        self.conv = CausalConv3d(self.channels, self.out_channels, kernel_size=kernel_size, bias=bias)

    def forward(self, x):
        return self.conv(x, up=self.upsample_factor)  # nearest upsample is address arithmetic in the padding pass


class DownsampleCausal3D(nn.Module):
    def __init__(self, channels, kernel_size=3, bias=True, stride=2):
        super().__init__()
        self.channels = self.out_channels = channels
        self.conv = CausalConv3d(channels, channels, kernel_size=kernel_size, stride=stride, bias=bias)

    def forward(self, x):
        return self.conv(x)


class ResnetBlockCausal3D(nn.Module):
    def __init__(self, *, in_channels, out_channels=None, dropout=0.0, groups=32, groups_out=None, pre_norm=True,
                 eps=1e-6, non_linearity="swish", output_scale_factor=1.0, use_in_shortcut=None,
                 conv_shortcut_bias=True, conv_3d_out_channels=None):
        super().__init__()
        out_channels = in_channels if out_channels is None else out_channels
        self.in_channels, self.out_channels = in_channels, out_channels
        self.output_scale_factor = output_scale_factor
        assert output_scale_factor == 1.0 and dropout == 0.0
        self.norm1 = nn.GroupNorm(groups, in_channels, eps=eps, affine=True)
        self.conv1 = CausalConv3d(in_channels, out_channels, kernel_size=3, stride=1)
        self.norm2 = nn.GroupNorm(groups_out or groups, out_channels, eps=eps, affine=True)
        c3 = conv_3d_out_channels or out_channels
        self.conv2 = CausalConv3d(out_channels, c3, kernel_size=3, stride=1)
        self.use_in_shortcut = in_channels != c3 if use_in_shortcut is None else use_in_shortcut
        self.conv_shortcut = CausalConv3d(in_channels, c3, kernel_size=1, stride=1, bias=conv_shortcut_bias) \
            if self.use_in_shortcut else None

    def forward(self, x):
        h = self.conv1(x, norm=self.norm1, silu=True)
        sc = x if self.conv_shortcut is None else self.conv_shortcut(x)
        return self.conv2(h, norm=self.norm2, silu=True, residual=sc)  # (shortcut + h) fused in the conv epilogue


class _MidAttention(nn.Module):
    """State-dict twin of the diffusers `Attention` the reference instantiates at unet_causal_3d_blocks.py:311-325
    (1 head of C dims, GroupNorm, bias, residual): group_norm, to_q, to_k, to_v, to_out.0."""

    def __init__(self, channels, groups, eps):
        super().__init__()
        self.group_norm = nn.GroupNorm(groups, channels, eps=eps, affine=True)
        self.to_q = nn.Linear(channels, channels)
        self.to_k = nn.Linear(channels, channels)
        self.to_v = nn.Linear(channels, channels)
        self.to_out = nn.ModuleList([nn.Linear(channels, channels), nn.Dropout(0.0)])
        self.native = False   # set by AutoencoderKLCausal3D.enable_native_attention: one osb_attn_frames call, no SDPA

    def forward(self, x):
        osb = _osb()
        nb, T, H, W, C = x.shape
        hw = H * W
        shard = _TemporalShard.group
        stats = osb.group_stats(x, self.group_norm.num_groups, self.group_norm.eps)
        if shard is not None:
            stats = _combine_group_stats(stats, T * hw * (C // self.group_norm.num_groups), self.group_norm.eps, shard)
        h = osb.vae_prep(x, stats=stats, gamma=self.group_norm.weight, beta=self.group_norm.bias,
                         groups=self.group_norm.num_groups, slack_bytes=0).view(nb * T * hw, C)
        q = osb.gemm(h, self.to_q.weight, self.to_q.bias).view(nb, 1, T * hw, C)
        k = osb.gemm(h, self.to_k.weight, self.to_k.bias).view(nb, 1, T * hw, C)
        v = osb.gemm(h, self.to_v.weight, self.to_v.bias).view(nb, 1, T * hw, C)
        first = 0
        if shard is not None:
            # frame-sharded: queries stay local; keys / values of ALL ranks' frames are gathered (latent resolution: C = 512
            # per token) and the causal prefix of local frame f ends at global frame first + f
            k, v, first = _gather_frames(k, v, T, hw, shard)
        # Frame-causal attention (prepare_causal_attention_mask, :52-60): frame f attends to frames <= f, so the
        # mask is never materialised.
        if self.native:
            # one osb_attn_frames launch (wgmma, head_dim 512): the mask is a predicate on (query frame, key) in the kernel
            o = osb.attn_frames(q[:, 0], k[:, 0], v[:, 0], frame_tokens=hw, q_frame0=first).unsqueeze(1)
        else:
            # the default: one un-masked SDPA per query frame over the key prefix.  LIBRARY kernel (torch SDPA, head_dim
            # 512), kept as the default until the native path has been measured against it on the benchmark's VAE leg.
            o = torch.empty_like(q)
            for f in range(T):
                keys = (first + f + 1) * hw
                o[:, :, f * hw:(f + 1) * hw] = torch.nn.functional.scaled_dot_product_attention(
                    q[:, :, f * hw:(f + 1) * hw], k[:, :, :keys], v[:, :, :keys])
        out = osb.gemm(o.view(nb * T * hw, C), self.to_out[0].weight, self.to_out[0].bias, epilogue=osb.EPI_BIAS_GATE_RES,
                       residual=x.reshape(nb * T * hw, C))
        return out.view(nb, T, H, W, C)


def _gather_frames(k, v, T: int, hw: int, group):
    """k, v [nb, 1, T*hw, C] of this rank's T frames -> the same for the frames of all ranks in rank (= frame) order, and
    the global index of this rank's first frame.  One all-gather of the frame counts, one var-len gather of k|v."""
    import torch.distributed as dist

    from opensora.acceleration.communications import gather_forward_split_backward_var_len

    P, r = dist.get_world_size(group), dist.get_rank(group)
    counts = [torch.zeros(1, dtype=torch.long, device=k.device) for _ in range(P)]
    dist.all_gather(counts, torch.tensor([T], dtype=torch.long, device=k.device), group=group)
    counts = [int(c) for c in counts]
    kv = torch.cat((k, v), dim=1)                                    # [nb, 2, T*hw, C]
    kv = gather_forward_split_backward_var_len(kv, 2, group, [c * hw for c in counts])
    return kv[:, :1], kv[:, 1:], sum(counts[:r])


class UNetMidBlockCausal3D(nn.Module):
    def __init__(self, in_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6, resnet_act_fn="swish", resnet_groups=32,
                 attn_groups=None, resnet_pre_norm=True, add_attention=True, attention_head_dim=1, output_scale_factor=1.0):
        super().__init__()
        self.add_attention = add_attention
        attn_groups = attn_groups or resnet_groups
        mk = lambda: ResnetBlockCausal3D(in_channels=in_channels, out_channels=in_channels, eps=resnet_eps,  # noqa: E731
                                         groups=resnet_groups, output_scale_factor=output_scale_factor)
        resnets, attentions = [mk()], []
        for _ in range(num_layers):
            attentions.append(_MidAttention(in_channels, attn_groups, resnet_eps) if add_attention else None)
            resnets.append(mk())
        self.attentions = nn.ModuleList(attentions)
        self.resnets = nn.ModuleList(resnets)

    def forward(self, x, attention_mask=None):
        x = self.resnets[0](x)
        for attn, resnet in zip(self.attentions, self.resnets[1:]):
            if attn is not None:
                x = attn(x)
            x = resnet(x)
        return x


class DownEncoderBlockCausal3D(nn.Module):
    def __init__(self, in_channels, out_channels, dropout=0.0, num_layers=1, resnet_eps=1e-6, resnet_act_fn="swish",
                 resnet_groups=32, resnet_pre_norm=True, output_scale_factor=1.0, add_downsample=True, downsample_stride=2):
        super().__init__()
        self.resnets = nn.ModuleList([
            ResnetBlockCausal3D(in_channels=in_channels if i == 0 else out_channels, out_channels=out_channels,
                                eps=resnet_eps, groups=resnet_groups, output_scale_factor=output_scale_factor)
            for i in range(num_layers)])
        self.downsamplers = nn.ModuleList([DownsampleCausal3D(out_channels, stride=downsample_stride)]) if add_downsample else None

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.downsamplers is not None:
            for d in self.downsamplers:
                x = d(x)
        return x


class UpDecoderBlockCausal3D(nn.Module):
    def __init__(self, in_channels, out_channels, resolution_idx=None, dropout=0.0, num_layers=1, resnet_eps=1e-6,
                 resnet_act_fn="swish", resnet_groups=32, resnet_pre_norm=True, output_scale_factor=1.0,
                 add_upsample=True, upsample_scale_factor=(2, 2, 2)):
        super().__init__()
        self.resnets = nn.ModuleList([
            ResnetBlockCausal3D(in_channels=in_channels if i == 0 else out_channels, out_channels=out_channels,
                                eps=resnet_eps, groups=resnet_groups, output_scale_factor=output_scale_factor)
            for i in range(num_layers)])
        self.upsamplers = nn.ModuleList([UpsampleCausal3D(out_channels, out_channels=out_channels,
                                                          upsample_factor=upsample_scale_factor)]) if add_upsample else None
        self.resolution_idx = resolution_idx

    def forward(self, x):
        for r in self.resnets:
            x = r(x)
        if self.upsamplers is not None:
            for u in self.upsamplers:
                x = u(x)
        return x
