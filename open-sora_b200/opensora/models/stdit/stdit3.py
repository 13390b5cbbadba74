"""STDiT3 (Open-Sora v1.2 denoiser) on the H100-native osb200 kernels.

Same class / module path / registry keys / state-dict keys as upstream
`opensora/models/stdit/stdit3.py` (witnessed in the reference tree only by `gradio/app.py:119-137`
and docs/report_0{1,2,3}.md — see SURVEY.md §8(a-S), Appendix A), so `STDiT3.from_pretrained(...)`,
`build_module({"type": "STDiT3-XL/2", ...}, MODELS)` and `model(x, timestep, y, mask=..., fps=...,
height=..., width=...)` keep working.  The nn.Modules below only HOLD parameters; every FLOP of the
forward runs in libosb200.so (wgmma GEMMs with fused bias/GELU/gate+residual epilogues, the
flash attention with fused QK-RMSNorm + RoPE, the LN+modulate row kernel).  There is no
CPU or eager fallback: calling forward on a non-CUDA / non-bf16 model raises.

Per block (SURVEY.md §8a-S `STDiT3Block.forward`), 10 launches:
  ln_modulate -> qkv GEMM (+bias, +QK-RMSNorm, +RoPE, stored as attention operand tiles) -> attention
  -> proj GEMM (+gate, +residual) -> q GEMM (operand tiles) -> cross attention (kv_lens) -> proj GEMM (+residual)
  -> ln_modulate -> fc1 GEMM (+GELU-tanh) -> fc2 GEMM (+gate, +residual)
The 2*depth kv_linear projections of the (block-invariant) text tokens are batched into one GEMM.
q / k / v never exist in token layout: the projection epilogue writes "head tiles" (include/osb200.h) that the
attention kernel loads with one bulk copy per tile.  Head sizes the tile path is not built for (anything but
64 / 72 / 128, or an odd head count) use the register-path kernel `osb_attn_short` on token-layout q / k / v.
"""
from __future__ import annotations

import math
import os
from dataclasses import asdict, dataclass

import torch
import torch.distributed as dist
import torch.nn as nn

from opensora.registry import MODELS


@dataclass
class STDiT3Config:
    input_size: tuple = (None, None, None)
    input_sq_size: int = 512
    in_channels: int = 4
    patch_size: tuple = (1, 2, 2)
    hidden_size: int = 1152
    depth: int = 28
    num_heads: int = 16
    mlp_ratio: float = 4.0
    class_dropout_prob: float = 0.1
    pred_sigma: bool = True
    drop_path: float = 0.0
    caption_channels: int = 4096
    model_max_length: int = 300
    qk_norm: bool = True
    enable_flash_attn: bool = True       # accepted for config compatibility; attention is always osb200's
    enable_layernorm_kernel: bool = True  # idem
    enable_sequence_parallelism: bool = False
    only_train_temporal: bool = False
    freeze_y_embedder: bool = False
    skip_y_embedder: bool = False

    @property
    def out_channels(self) -> int:
        return self.in_channels * 2 if self.pred_sigma else self.in_channels


# ---------------------------------------------------------------------------------------------
# parameter containers (state-dict layout of SURVEY.md Appendix A "Module tree")
# ---------------------------------------------------------------------------------------------
class _Mlp(nn.Module):
    def __init__(self, din, dh, dout=None):
        super().__init__()
        self.fc1 = nn.Linear(din, dh)
        self.fc2 = nn.Linear(dh, dout or din)


class _Embedder(nn.Module):  # t_embedder / fps_embedder: mlp.0, mlp.2
    def __init__(self, hidden, freq=256):
        super().__init__()
        self.frequency_embedding_size = freq
        self.mlp = nn.Sequential(nn.Linear(freq, hidden), nn.SiLU(), nn.Linear(hidden, hidden))


class _Caption(nn.Module):
    def __init__(self, cin, hidden, tokens):
        super().__init__()
        self.y_proj = _Mlp(cin, hidden, hidden)
        self.register_buffer("y_embedding", torch.randn(tokens, cin) / cin**0.5)


class _Norm(nn.Module):
    def __init__(self, d):
        super().__init__()
        self.weight = nn.Parameter(torch.ones(d))


class _Attn(nn.Module):
    def __init__(self, dim, heads, qk_norm):
        super().__init__()
        self.qkv = nn.Linear(dim, 3 * dim)
        self.q_norm = _Norm(dim // heads) if qk_norm else nn.Identity()
        self.k_norm = _Norm(dim // heads) if qk_norm else nn.Identity()
        self.proj = nn.Linear(dim, dim)


class _Cross(nn.Module):
    def __init__(self, dim):
        super().__init__()
        self.q_linear = nn.Linear(dim, dim)
        self.kv_linear = nn.Linear(dim, 2 * dim)
        self.proj = nn.Linear(dim, dim)


class STDiT3Block(nn.Module):
    def __init__(self, hidden, heads, mlp_ratio, qk_norm, temporal):
        super().__init__()
        self.temporal = temporal
        self.attn = _Attn(hidden, heads, qk_norm)
        self.cross_attn = _Cross(hidden)
        self.mlp = _Mlp(hidden, int(hidden * mlp_ratio))
        self.scale_shift_table = nn.Parameter(torch.randn(6, hidden) / hidden**0.5)


class _Final(nn.Module):
    def __init__(self, hidden, num_patch, cout):
        super().__init__()
        self.linear = nn.Linear(hidden, num_patch * cout)
        self.scale_shift_table = nn.Parameter(torch.randn(2, hidden) / hidden**0.5)


class _PatchEmbed(nn.Module):
    def __init__(self, patch, cin, hidden):
        super().__init__()
        self.patch_size = patch
        self.proj = nn.Conv3d(cin, hidden, kernel_size=patch, stride=patch)  # parameter container only


def _timestep_embedding(t, dim, max_period=10000):
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


class STDiT3(nn.Module):
    config_class = STDiT3Config

    def __init__(self, config: STDiT3Config | None = None, **kwargs):
        super().__init__()
        if config is None:
            config = STDiT3Config(**kwargs)
        c = self.config = config
        self.hidden_size, self.num_heads, self.depth = c.hidden_size, c.num_heads, c.depth
        self.head_dim = c.hidden_size // c.num_heads
        self.patch_size = tuple(c.patch_size)
        self.in_channels, self.out_channels = c.in_channels, c.out_channels
        self.input_sq_size = c.input_sq_size
        self.x_embedder = _PatchEmbed(self.patch_size, c.in_channels, c.hidden_size)
        self.t_embedder = _Embedder(c.hidden_size)
        self.fps_embedder = _Embedder(c.hidden_size)
        self.t_block = nn.Sequential(nn.SiLU(), nn.Linear(c.hidden_size, 6 * c.hidden_size))
        self.y_embedder = _Caption(c.caption_channels, c.hidden_size, c.model_max_length)
        self.spatial_blocks = nn.ModuleList(
            [STDiT3Block(c.hidden_size, c.num_heads, c.mlp_ratio, c.qk_norm, False) for _ in range(c.depth)])
        self.temporal_blocks = nn.ModuleList(
            [STDiT3Block(c.hidden_size, c.num_heads, c.mlp_ratio, c.qk_norm, True) for _ in range(c.depth)])
        self.final_layer = _Final(c.hidden_size, math.prod(self.patch_size), c.out_channels)
        self._cache: dict = {}
        self._sp_group = None
        self._peer = None
        self._sp_exchange = "nccl"
        self._sp_config_checked = False
        self.register_load_state_dict_post_hook(lambda m, k: m._cache.clear())

    # ---- construction helpers ---------------------------------------------------------------
    @classmethod
    def from_pretrained(cls, path: str | None = None, **kwargs):
        """`STDiT3.from_pretrained(weight_path, **model_kwargs)` (gradio/app.py:124): local directory or
        file holding `model.safetensors` / a torch state dict.  No hub download (no network)."""
        cfg_kw = {}
        if path and os.path.isdir(path) and os.path.exists(os.path.join(path, "config.json")):
            import json

            with open(os.path.join(path, "config.json")) as fh:   # the checkpoint's own architecture, overridden by kwargs
                cfg_kw = {k: (tuple(v) if isinstance(v, list) else v) for k, v in json.load(fh).items()
                          if k in STDiT3Config.__dataclass_fields__}
        cfg_kw.update({k: v for k, v in kwargs.items() if k in STDiT3Config.__dataclass_fields__})
        model = cls(STDiT3Config(**cfg_kw))
        if path:
            f = path
            if os.path.isdir(path):
                for cand in ("model.safetensors", "diffusion_pytorch_model.safetensors", "model.pt", "pytorch_model.bin"):
                    if os.path.exists(os.path.join(path, cand)):
                        f = os.path.join(path, cand)
                        break
            if f.endswith(".safetensors"):
                from safetensors.torch import load_file

                sd = load_file(f)
            else:
                sd = torch.load(f, map_location="cpu")
            res = model.load_state_dict(sd, strict=False)
            # y_embedding is a buffer older checkpoints may lack; anything else missing or unexpected means the file does
            # not belong to this architecture and the model would silently keep random weights
            missing = [k for k in res.missing_keys if k != "y_embedder.y_embedding"]
            if missing or res.unexpected_keys:
                raise RuntimeError(f"{f}: state dict does not match STDiT3 ({len(missing)} missing, e.g. {missing[:3]}; "
                                   f"{len(res.unexpected_keys)} unexpected, e.g. {list(res.unexpected_keys)[:3]})")
        return model

    def _apply(self, fn, *a, **k):  # .to()/.cuda()/.bfloat16() invalidate the packed-weight cache
        self._cache = {}
        return super()._apply(fn, *a, **k)

    def _configured_sp_group(self):
        """Upstream's switch: `enable_sequence_parallelism=True` in the config + the group registered with
        `opensora.acceleration.parallel_states.set_sequence_parallel_group` (parallel_states.py:18-23)."""
        if self._sp_group is None and self.config.enable_sequence_parallelism and not self._sp_config_checked:
            from opensora.acceleration.parallel_states import get_sequence_parallel_group

            self._sp_config_checked = True
            group = get_sequence_parallel_group()
            if group is not None and dist.is_initialized() and dist.get_world_size(group) > 1:
                self.enable_sequence_parallel(group)
        return self._sp_group

    def enable_sequence_parallel(self, group, exchange: str | None = None) -> None:
        """Shard tokens over `group` (SURVEY.md §8e): T-sharded for spatial / cross / MLP, transposed to
        S-sharded around each temporal attention.  `exchange`: "peer" = the producing kernels store straight into the
        consuming rank's buffer over NVLink (opensora/acceleration/peer_exchange.py; default on CUDA), "nccl" = one
        all_to_all_single per transposition (opensora/acceleration/communications.py; the only choice on gloo / CPU)."""
        self._sp_group = group
        self._cache = {}
        self._peer = None
        self._sp_exchange = exchange or os.environ.get("OSB_SP_EXCHANGE", "peer")

    @property
    def sp_exchange_kind(self) -> str:
        if self._sp_group is None:
            return "none"
        return ("peer stores from the producing kernels (symmetric memory over NVLink) + osb_comm_barrier"
                if getattr(self, "_peer", None) is not None else "nccl all_to_all_single")

    def _peer_exchange(self, dev):
        """The PeerExchange of this model (created collectively on first use), or None when the exchange is NCCL's."""
        if self._sp_group is None or self._sp_exchange != "peer" or dev.type != "cuda" or not self._use_tiles():
            return None
        if self._peer is None:
            try:
                from opensora.acceleration.peer_exchange import PeerExchange

                self._peer = PeerExchange(self._sp_group, dev)
            except Exception as e:   # no symmetric memory on this system: the collective path is still correct
                import warnings

                warnings.warn(f"peer-memory exchange unavailable ({e!r}); using NCCL all_to_all")
                self._sp_exchange = "nccl"
                return None
        return self._peer

    # ---- CUDA-graph replay of one step (fixed shapes): removes the ~600 Python-issued launches from the critical
    # path.  Matters when the per-rank work is small (sequence parallel at 8 GPUs is host-bound otherwise). ----------
    def capture(self, x, timestep, y, mask=None, x_mask=None, fps=None, height=None, width=None):
        """Capture `forward` on static device copies of the inputs; returns a `replay(x, timestep, y, mask, fps)`
        callable that copies new values into the static buffers and replays the graph.  `height` / `width` must be
        host values (they only select the cached positional table)."""
        dev = self.x_embedder.proj.weight.device
        st = dict(x=x.to(dev).clone(), timestep=timestep.to(dev).clone(), y=y.to(dev).clone(),
                  mask=None if mask is None else mask.to(dev).clone(), fps=fps.to(dev).clone(),
                  x_mask=None if x_mask is None else x_mask.to(dev).clone())
        hw = dict(height=[float(height[0])], width=[float(width[0])])
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.cuda.stream(side), torch.no_grad():
            for _ in range(2):  # warm-up outside capture: library init, cached tables, allocator pools, NCCL channels
                self.forward(**st, **hw)
        torch.cuda.current_stream(dev).wait_stream(side)
        import osb200

        graph = torch.cuda.CUDAGraph()
        l0 = osb200.launch_count()
        with torch.cuda.graph(graph), torch.no_grad():
            out = self.forward(**st, **hw)
        kernels = osb200.launch_count() - l0   # osb200 kernels one replay re-issues

        def replay(x, timestep, y, mask=None, fps=None, x_mask=None, **_):
            st["x"].copy_(x, non_blocking=True)
            st["timestep"].copy_(timestep, non_blocking=True)
            st["y"].copy_(y, non_blocking=True)
            if mask is not None and st["mask"] is not None:
                st["mask"].copy_(mask, non_blocking=True)
            if fps is not None:
                st["fps"].copy_(fps, non_blocking=True)
            if x_mask is not None and st["x_mask"] is not None:
                st["x_mask"].copy_(x_mask, non_blocking=True)
            graph.replay()
            return out

        replay.graph = graph
        replay.kernel_launches = kernels
        return replay

    def get_dynamic_size(self, x):
        _, _, T, H, W = x.size()
        pt, ph, pw = self.patch_size
        return -(-T // pt), -(-H // ph), -(-W // pw)

    # ---- cached per-model constants ------------------------------------------------------------
    def _const(self, dev):
        key = ("const", dev)
        if key in self._cache:
            return self._cache[key]
        blocks = [b for pair in zip(self.spatial_blocks, self.temporal_blocks) for b in pair]
        d = {}
        # all 2*depth kv_linear weights of the cross-attentions in one [2*depth*2C, C] matrix
        d["kv_w"] = torch.cat([b.cross_attn.kv_linear.weight for b in blocks], 0).contiguous()
        d["kv_b"] = torch.cat([b.cross_attn.kv_linear.bias for b in blocks], 0).contiguous()
        d["tables"] = torch.stack([b.scale_shift_table for b in blocks], 0).float()  # [2*depth, 6, C]
        d["final_table"] = self.final_layer.scale_shift_table.float()
        pt, ph, pw = self.patch_size
        d["x_w"] = self.x_embedder.proj.weight.reshape(self.hidden_size, -1).contiguous()  # [C, Cin*pt*ph*pw]
        half = self.head_dim // 2 * 2
        inv = 1.0 / (10000.0 ** (torch.arange(0, half, 2, device=dev).float() / self.head_dim))
        d["rope_inv"] = inv
        self._cache[key] = d
        return d

    def _rope(self, T, dev):
        key = ("rope", T, dev)
        if key not in self._cache:
            ang = torch.arange(T, device=dev, dtype=torch.float32)[:, None] * self._const(dev)["rope_inv"][None]
            self._cache[key] = (ang.cos().contiguous(), ang.sin().contiguous())
        return self._cache[key]

    def _pos_embed(self, H, W, scale, base_size, dev):
        key = ("pos", H, W, round(scale, 6), base_size, dev)
        if key not in self._cache:
            half = self.hidden_size // 2
            inv = 1.0 / (10000 ** (torch.arange(0, half, 2, device=dev).float() / half))
            gh = torch.arange(H, device=dev) / scale * (base_size / H)
            gw = torch.arange(W, device=dev) / scale * (base_size / W)
            gh, gw = torch.meshgrid(gw, gh, indexing="ij")
            gh, gw = gh.t().reshape(-1), gw.t().reshape(-1)

            def sc(t):
                o = torch.einsum("i,d->id", t, inv)
                return torch.cat((torch.sin(o), torch.cos(o)), dim=-1)

            self._cache[key] = torch.cat([sc(gh), sc(gw)], dim=-1).to(torch.bfloat16)  # [S, C]
        return self._cache[key]

    # ---- forward ---------------------------------------------------------------------------------
    def forward(self, x, timestep, y, mask=None, x_mask=None, fps=None, height=None, width=None, **kwargs):
        import osb200 as osb

        w0 = self.x_embedder.proj.weight
        osb.require_cuda_bf16(w0, "STDiT3")
        dev = w0.device
        bf = torch.bfloat16
        C, Hh, D = self.hidden_size, self.num_heads, self.head_dim
        cst = self._const(dev)
        B = x.size(0)
        x = x.to(dev, bf)
        _, Cin, Tx, Hx, Wx = x.shape
        pt, ph, pw = self.patch_size
        if Tx % pt or Hx % ph or Wx % pw:
            x = torch.nn.functional.pad(x, (0, -Wx % pw, 0, -Hx % ph, 0, -Tx % pt))
        T, H, W = self.get_dynamic_size(x)
        S = H * W
        # sequence parallelism (SURVEY.md §8e): this rank owns frames [t0, t0+Tl) for every token-local op
        sp = self._configured_sp_group()
        P = dist.get_world_size(sp) if sp is not None else 1
        if P > 1:
            if T % P or S % P:
                raise ValueError(f"sequence parallel needs T ({T}) and S ({S}) divisible by the group size {P}")
            Tl = T // P
            t0 = dist.get_rank(sp) * Tl
            x = x[:, :, t0 * pt:(t0 + Tl) * pt]
            if x_mask is not None:
                x_mask = x_mask.reshape(B, T)[:, t0:t0 + Tl]
        else:
            Tl = T
        N = Tl * S  # local tokens per sample
        scale = (float(height[0]) * float(width[0])) ** 0.5 / self.input_sq_size
        pos = self._pos_embed(H, W, scale, round(S**0.5), dev)

        # ---- conditioning vectors (tiny: M = B rows) --------------------------------------------
        def emb(e, v, cast_input):
            # upstream casts `timestep` to the model dtype BEFORE the sinusoidal embedding (x, timestep, y = .to(dtype);
            # oracle/stdit3_oracle.py forward): 537 becomes 536 in bf16.  fps is embedded at full precision.
            v = v.to(dev)
            v = v.to(bf).float() if cast_input else v.float()
            f = _timestep_embedding(v.reshape(-1), e.frequency_embedding_size).to(bf)
            h = osb.gemm(f, e.mlp[0].weight, e.mlp[0].bias)
            return osb.gemm(torch.nn.functional.silu(h), e.mlp[2].weight, e.mlp[2].bias)

        fps_e = emb(self.fps_embedder, fps, False)
        if fps_e.shape[0] != B:
            fps_e = fps_e.repeat(B // fps_e.shape[0], 1)
        ts = [timestep] + ([torch.zeros_like(timestep)] if x_mask is not None else [])
        t_all = torch.cat([emb(self.t_embedder, t_, True) + fps_e for t_ in ts], 0)            # [B or 2B, C]
        t_mlp = osb.gemm(torch.nn.functional.silu(t_all), self.t_block[1].weight, self.t_block[1].bias)  # [., 6C]
        nb = 2 * self.depth
        # modulation for every block at once: [B', nb, 6, C] fp32  (table + t), App. A "Modulation"
        mod = (cst["tables"][None] + t_mlp.float().view(-1, 1, 6, C)).contiguous()
        fmod = (cst["final_table"][None] + t_all.float()[:, None]).contiguous()         # [B', 2, C]
        mod_index = None
        group_rows = N
        if x_mask is not None:
            xm = x_mask.to(dev).bool().reshape(B, Tl)
            base = torch.arange(B, device=dev, dtype=torch.int32)[:, None]
            mod_index = torch.where(xm, base, base + B).to(torch.int32).reshape(-1).contiguous()
            group_rows = S

        # ---- text tokens: y_embedder MLP, then every block's kv_linear in one GEMM -------------------
        Ly = y.shape[-2]
        yt = y.to(dev, bf).reshape(-1, y.shape[-1])
        if yt.shape[0] != B * Ly:
            raise ValueError("y must be [B, 1, L, caption_channels]")
        yp = self.y_embedder.y_proj
        yh = osb.gemm(yt, yp.fc1.weight, yp.fc1.bias, epilogue=osb.EPI_BIAS_GELU_TANH)
        ye = osb.gemm(yh, yp.fc2.weight, yp.fc2.bias)                                    # [B*Ly, C]
        use_tiles = self._use_tiles()
        if use_tiles:   # keys / values of all 2*depth blocks as attention operand tiles: [block][k|v][head][tile]
            kv_all = self._tiles(osb, ("kv", B, Ly), B * Ly, osb.tile_map(0, Ly, keys_only=True), 2 * nb, dev)
            osb.gemm_head_tiles(ye, cst["kv_w"], cst["kv_b"], kv_all, nkinds=2)
        else:
            kv_all = osb.gemm(ye, cst["kv_w"], cst["kv_b"])                              # [B*Ly, nb*2C]
        if mask is not None:
            m2 = mask.to(dev)
            if m2.shape[0] != B:
                m2 = m2.repeat(B // m2.shape[0], 1)
            kv_lens = m2.reshape(B, -1).ne(0).sum(dim=1).to(torch.int32).contiguous()
        else:
            kv_lens = None

        # ---- patch embedding (conv with kernel == stride  ==  GEMM over patch vectors) + pos_embed ---
        xp = x.reshape(B, Cin, Tl, pt, H, ph, W, pw).permute(0, 2, 4, 6, 1, 3, 5, 7).reshape(B * N, Cin * pt * ph * pw)
        Kp = xp.shape[1]
        if Kp % 8:
            xp = torch.nn.functional.pad(xp, (0, -Kp % 8))
            xw = torch.nn.functional.pad(cst["x_w"], (0, -Kp % 8))
        else:
            xw = cst["x_w"]
        xs = osb.gemm(xp.contiguous(), xw, self.x_embedder.proj.bias)                    # [B*N, C]
        xs = (xs.view(B * Tl, S, C) + pos[None]).view(B * N, C)

        # ---- workspaces reused by every block ------------------------------------------------------
        R = B * N

        def wsbuf(name, *shape):   # block workspaces live with the model (no allocator traffic per step, graph-safe)
            key = ("ws", name, shape, dev)
            if key not in self._cache:
                self._cache[key] = torch.empty(*shape, dtype=bf, device=dev)
            return self._cache[key]

        xm_buf = wsbuf("xm", R, C)
        ao = wsbuf("ao", R, C)
        hid = wsbuf("hid", R, int(C * self.config.mlp_ratio))
        cos, sin = self._rope(T, dev)
        ws = dict(xm=xm_buf, ao=ao, hid=hid, cos=cos, sin=sin, kv=kv_all, kv_lens=kv_lens, tiles=use_tiles,
                  peer=self._peer_exchange(dev) if P > 1 else None)
        if use_tiles:
            Sl = S // P   # temporal attention runs on this rank's S/P columns of every frame
            ws["sp_t"] = self._tiles(osb, ("spatial", B, Tl, S), R, osb.tile_map(0, S), 3, dev)
            # temporal attention tiles.  Default: LN+modulate writes its rows transposed to [B, S, T] (a free row
            # permutation of its stores), so a temporal sequence is a contiguous row block for the QKV GEMM (tile map mode 0)
            # and only the attention OUTPUT is addressed frame-major (`tm_out`, mode 1).  When the rows arrive frame-major
            # (NCCL all-to-all exchange) the GEMM reads them through a strided TMA view instead (mode 1 map).
            ws["tm_out"] = osb.tile_map(1, T, Sl, T)
            ws["tm_t"] = self._tiles(osb, ("temporal", B, T, Sl), B * T * Sl, osb.tile_map(0, T), 3, dev)
            ws["xm_t"] = wsbuf("xm_t", R, C) if P == 1 else None
            ws["q_t"] = self._tiles(osb, ("crossq", B, N), R, osb.tile_map(0, N, pack=False), 1, dev)
        else:
            ws["qkv"] = wsbuf("qkv", R, 3 * C)
            ws["qc"] = wsbuf("qc", R, C)

        bi = 0
        for sb, tb in zip(self.spatial_blocks, self.temporal_blocks):
            for blk in (sb, tb):
                m = mod[:, bi]  # [B', 6, C] view, row stride = mod.stride(0)
                self._block(osb, blk, bi, xs, m, mod_index, group_rows, Ly, B, T, Tl, S, ws, sp if P > 1 else None)
                bi += 1

        # ---- final layer + unpatchify -----------------------------------------------------------------
        osb.ln_modulate(xs, fmod[:, 0], fmod[:, 1], group_rows=group_rows, mod_index=mod_index, out=xm_buf)
        fl = self.final_layer.linear
        o = osb.gemm(xm_buf, fl.weight, fl.bias)                                         # [B*N, pt*ph*pw*Cout]
        if P > 1:  # exit all-gather of the T shards (communications.py gather_forward_split_backward)
            from opensora.acceleration.communications import gather_forward_split_backward

            o = gather_forward_split_backward(o.view(B, Tl, S, -1), sp, dim=1).reshape(B * T * S, -1)
        return self._unpatchify(o, B, T, H, W, Tx, Hx, Wx)

    def _unpatchify(self, o, B, T, H, W, Tx, Hx, Wx):
        pt, ph, pw = self.patch_size
        o = o.view(B, T, H, W, pt, ph, pw, self.out_channels).permute(0, 7, 1, 4, 2, 5, 3, 6)
        o = o.reshape(B, self.out_channels, T * pt, H * ph, W * pw)[:, :, :Tx, :Hx, :Wx]
        return o.to(torch.float32)

    def _use_tiles(self) -> bool:
        """The head-tile attention path (osb_gemm_head_tiles + osb_attn_tiles) is built for head sizes 64 / 72 / 128 and an
        even head count; OSB_ATTN_TILES=0 forces the register-path kernel (A/B measurements)."""
        return (self.head_dim in (64, 72, 128) and self.num_heads % 2 == 0
                and os.environ.get("OSB_ATTN_TILES", "1") != "0")

    def _tiles(self, osb, key, rows, tmap, kinds, dev):
        """Tile workspaces are cached per shape: they are zero-filled once (rows no token maps to must stay finite)."""
        key = ("tiles", key, tmap.key(), kinds, dev)
        if key not in self._cache:
            self._cache[key] = osb.HeadTiles(rows, tmap, kinds, self.num_heads, self.head_dim, dev)
        return self._cache[key]

    def _block(self, osb, blk, bi, xs, m, mod_index, group_rows, Ly, B, T, Tl, S, ws, sp):
        C, Hh, D = self.hidden_size, self.num_heads, self.head_dim
        N = Tl * S
        a, ca, mlp = blk.attn, blk.cross_attn, blk.mlp
        qn = a.q_norm.weight if isinstance(a.q_norm, _Norm) else None
        kn = a.k_norm.weight if isinstance(a.k_norm, _Norm) else None
        xm_buf, ao, hid, cos, sin, tiles = ws["xm"], ws["ao"], ws["hid"], ws["cos"], ws["sin"], ws["tiles"]
        # 1. self attention (spatial: sequences over S; temporal: sequences over T with RoPE)
        peer = ws.get("peer") if (blk.temporal and sp is not None) else None
        if peer is not None:
            # sequence parallel, peer-memory exchange: LN+modulate stores every row into the xt buffer of the rank that
            # owns its S-column, the attention epilogue stores every output row into the ao buffer of the rank that owns
            # its frame; one barrier kernel after each producer.  Rows stay B*T*S/P on both sides.
            Sl = S // (T // Tl)
            xt, xt_ptrs = peer.buffer("xt", B * Sl * T, C)
            ar, ar_ptrs = peer.buffer("ao", B * N, C)
            osb.ln_modulate(xs, m[:, 0], m[:, 1], group_rows=group_rows, mod_index=mod_index,
                            scatter=peer.scatter(4, Tl, S, xt_ptrs))     # -> [B, S/P, T] on the rank that owns the column
            peer.barrier()
            tt = ws["tm_t"]
            osb.gemm_head_tiles(xt, a.qkv.weight, a.qkv.bias, tt, nkinds=3, norm_w=(qn, kn, None), rope=(cos, sin),
                                rope_kinds=0b011)
            osb.attn_tiles(tt, tt, None, Lk=T, num_seqs=B * Sl, out_map=ws["tm_out"],
                           out_scatter=peer.scatter(2, T, Sl, ar_ptrs), out_ld=C)
            peer.barrier()
            ao = ar
        elif blk.temporal and tiles and sp is None:
            # single GPU: LN+modulate stores its rows transposed ([B, T, S] -> [B, S, T]) so temporal sequences are
            # contiguous row blocks; the attention output comes back frame-major
            xm_t, tt = ws["xm_t"], ws["tm_t"]
            osb.ln_modulate(xs, m[:, 0], m[:, 1], group_rows=group_rows, mod_index=mod_index,
                            scatter=osb.make_scatter(3, 1, 0, T, S, [xm_t]))
            osb.gemm_head_tiles(xm_t, a.qkv.weight, a.qkv.bias, tt, nkinds=3, norm_w=(qn, kn, None), rope=(cos, sin),
                                rope_kinds=0b011)
            osb.attn_tiles(tt, tt, ao, Lk=T, num_seqs=B * S, out_map=ws["tm_out"])
        elif blk.temporal:
            osb.ln_modulate(xs, m[:, 0], m[:, 1], group_rows=group_rows, mod_index=mod_index, out=xm_buf)
            if sp is not None:
                # T-sharded -> S-sharded transposition (all-to-all over NVLink), attention over the full T
                # for this rank's S/P columns, and back.  Rows stay B*T*S/P on both sides.
                from opensora.acceleration.communications import all_to_all

                Sl = S // (T // Tl)
                xt = all_to_all(xm_buf.view(B, Tl, S, C), sp, scatter_dim=2, gather_dim=1).view(B * T * Sl, C)
            else:
                Sl, xt = S, xm_buf
            ao_t = ao if sp is None else torch.empty_like(ao)
            if tiles:
                # (looked up here, not through a closure stored in `ws`: a ws -> lambda -> ws cycle would keep every
                # forward's workspaces alive until the cyclic GC runs, and the allocator would cudaMalloc new ones each step)
                tt = self._tiles(osb, ("temporal-fm", B, T, Sl), B * T * Sl, ws["tm_out"], 3, xs.device)
                osb.gemm_head_tiles(xt, a.qkv.weight, a.qkv.bias, tt, nkinds=3, norm_w=(qn, kn, None), rope=(cos, sin),
                                    rope_kinds=0b011)
                osb.attn_tiles(tt, tt, ao_t, Lk=T, num_seqs=B * Sl)
            else:
                qkv = ws["qkv"]
                osb.gemm(xt, a.qkv.weight, a.qkv.bias, out=qkv)
                strides = (T * Sl, 1, Sl)
                osb.attn_short(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ao_t, num_seqs=B * Sl, seqs_per_batch=Sl,
                               q_strides=strides, k_strides=strides, Lq=T, Lk=T, num_heads=Hh, head_dim=D,
                               q_norm_w=qn, k_norm_w=kn, rope_cos=cos, rope_sin=sin)
            if sp is not None:
                ao = all_to_all(ao_t.view(B, T, Sl, C), sp, scatter_dim=1, gather_dim=2).view(B * N, C)
        elif tiles:
            osb.ln_modulate(xs, m[:, 0], m[:, 1], group_rows=group_rows, mod_index=mod_index, out=xm_buf)
            st = ws["sp_t"]
            osb.gemm_head_tiles(xm_buf, a.qkv.weight, a.qkv.bias, st, nkinds=3, norm_w=(qn, kn, None))
            osb.attn_tiles(st, st, ao, Lk=S, num_seqs=B * Tl)
        else:
            osb.ln_modulate(xs, m[:, 0], m[:, 1], group_rows=group_rows, mod_index=mod_index, out=xm_buf)
            qkv = ws["qkv"]
            osb.gemm(xm_buf, a.qkv.weight, a.qkv.bias, out=qkv)
            strides = (N, S, 1)
            osb.attn_short(qkv[:, :C], qkv[:, C:2 * C], qkv[:, 2 * C:], ao, num_seqs=B * Tl, seqs_per_batch=Tl,
                           q_strides=strides, k_strides=strides, Lq=S, Lk=S, num_heads=Hh, head_dim=D,
                           q_norm_w=qn, k_norm_w=kn)
        osb.gemm(ao, a.proj.weight, a.proj.bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=xs, gate=m[:, 2],
                 group_rows=group_rows, mod_index=mod_index, out=xs)
        # 2. cross attention over the T5 tokens (plain residual)
        ao = ws["ao"]
        if tiles:
            qt = ws["q_t"]
            osb.gemm_head_tiles(xs, ca.q_linear.weight, ca.q_linear.bias, qt, nkinds=1)
            osb.attn_tiles(qt, ws["kv"], ao, q_kind=0, k_kind=2 * bi, v_kind=2 * bi + 1, Lk=Ly, num_seqs=B,
                           kv_lens=ws["kv_lens"])
        else:
            qc = ws["qc"]
            kv = ws["kv"][:, bi * 2 * C:(bi + 1) * 2 * C]
            osb.gemm(xs, ca.q_linear.weight, ca.q_linear.bias, out=qc)
            osb.attn_short(qc, kv[:, :C], kv[:, C:], ao, num_seqs=B, seqs_per_batch=1, q_strides=(N, 0, 1),
                           k_strides=(Ly, 0, 1), Lq=N, Lk=Ly, num_heads=Hh, head_dim=D, kv_lens=ws["kv_lens"])
        osb.gemm(ao, ca.proj.weight, ca.proj.bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=xs, gate=None, out=xs)
        # 3. MLP
        osb.ln_modulate(xs, m[:, 3], m[:, 4], group_rows=group_rows, mod_index=mod_index, out=xm_buf)
        osb.gemm(xm_buf, mlp.fc1.weight, mlp.fc1.bias, epilogue=osb.EPI_BIAS_GELU_TANH, out=hid)
        osb.gemm(hid, mlp.fc2.weight, mlp.fc2.bias, epilogue=osb.EPI_BIAS_GATE_RES, residual=xs, gate=m[:, 5],
                 group_rows=group_rows, mod_index=mod_index, out=xs)


def _build(from_pretrained=None, **kwargs):
    kwargs.pop("force_huggingface", None)
    if from_pretrained:
        return STDiT3.from_pretrained(from_pretrained, **kwargs)
    fields = STDiT3Config.__dataclass_fields__
    return STDiT3(STDiT3Config(**{k: v for k, v in kwargs.items() if k in fields}))


@MODELS.register_module("STDiT3-XL/2")
def STDiT3_XL_2(from_pretrained=None, **kwargs):
    return _build(from_pretrained, **{**dict(depth=28, hidden_size=1152, patch_size=(1, 2, 2), num_heads=16), **kwargs})


@MODELS.register_module("STDiT3-3B/2")
def STDiT3_3B_2(from_pretrained=None, **kwargs):
    return _build(from_pretrained, **{**dict(depth=28, hidden_size=1872, patch_size=(1, 2, 2), num_heads=26), **kwargs})


@MODELS.register_module("STDiT3-XS/2")
def STDiT3_XS_2(from_pretrained=None, **kwargs):
    """Builder-defined plumbing size of BASELINE.json configs[0] (no upstream equivalent)."""
    return _build(from_pretrained, **{**dict(depth=2, hidden_size=288, patch_size=(1, 2, 2), num_heads=4), **kwargs})
