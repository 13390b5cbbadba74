"""Native mid-block attention of the causal VAE on the CPU (`-m "not gpu"`): the stand-in's `attn_frames` against an
explicit-mask fp32 softmax built from the oracle's `causal_mask` (the pinned restatement of the reference's
`prepare_causal_attention_mask`), and the host side of `AutoencoderKLCausal3D.enable_native_attention()` on a small VAE
whose mid block is 512 wide: same result as the SDPA path within the bf16 bar, one launch instead of T SDPA calls,
untiled, tiled and frame-sharded, the refusal on another width, and the layout of the C args struct."""
import os

import pytest
import torch

from tests import fake_osb200_attn_frames as FA
from tests.util import rel_l2

BAR = 4e-3          # the bf16 attention bar of the GPU tests
VAE_BAR = 1.5e-2    # the bar of the other whole-model VAE comparisons in bf16


@pytest.fixture
def fake_frames(fake_osb, monkeypatch):
    FA.install(monkeypatch)
    return fake_osb


def masked_softmax_reference(q, k, v, hw, q_frame0=0):
    """fp32, the reference's way: a dense 0 / -inf mask added to the scaled scores."""
    from oracle.vae_oracle import causal_mask

    Lq, Lk = q.shape[1], k.shape[1]
    frames = q_frame0 + -(-max(Lq, Lk) // hw) + 1
    mask = causal_mask(frames, hw, q.device, torch.float32)[q_frame0 * hw:q_frame0 * hw + Lq, :Lk]
    s = q.float() @ k.float().transpose(1, 2) * q.shape[-1] ** -0.5 + mask[None]
    return torch.softmax(s, -1) @ v.float()


@pytest.mark.parametrize("hw", [1, 4, 100])
@pytest.mark.parametrize("T", [1, 3, 5])
def test_stand_in_matches_the_explicit_mask(fake_frames, hw, T):
    torch.manual_seed(hw * 10 + T)
    q, k, v = (torch.randn(2, T * hw, 512).to(torch.bfloat16) for _ in range(3))
    out = fake_frames.attn_frames(q, k, v, frame_tokens=hw)
    assert out.shape == q.shape and out.dtype == torch.bfloat16
    assert rel_l2(out, masked_softmax_reference(q, k, v, hw)) < BAR
    assert [c[0] for c in fake_frames.calls] == ["attn_frames"] and fake_frames.launch_count() == 1


def test_stand_in_with_a_frame_offset_and_column_slices(fake_frames):
    """Frame-sharded shape: 2 local frames starting at global frame 2, keys of 5 frames; q | k | v as column slices of
    one buffer (ld 1536) and a batch of 2."""
    torch.manual_seed(5)
    hw, Tq, Tk, first = 4, 2, 5, 2
    buf = torch.randn(2, Tk * hw, 1536).to(torch.bfloat16)
    q, k, v = buf[:, first * hw:(first + Tq) * hw, :512], buf[:, :, 512:1024], buf[:, :, 1024:]
    out = fake_frames.attn_frames(q, k, v, frame_tokens=hw, q_frame0=first)
    assert rel_l2(out, masked_softmax_reference(q, k, v, hw, first)) < BAR
    # local frames are global frames 2 and 3: changing the keys of frame 3 leaves the first local frame alone
    k2, v2 = k.clone(), v.clone()
    k2[:, 3 * hw:4 * hw] += 1
    v2[:, 3 * hw:4 * hw] += 1
    out2 = fake_frames.attn_frames(q, k2, v2, frame_tokens=hw, q_frame0=first)
    assert torch.equal(out2[:, :hw], out[:, :hw]) and not torch.equal(out2[:, hw:], out[:, hw:])


def test_stand_in_refusals_count_no_launch(fake_frames):
    q = torch.zeros(1, 8, 512, dtype=torch.bfloat16)
    for kw, args in ((dict(frame_tokens=0), (q, q, q)), (dict(frame_tokens=4, q_frame0=-1), (q, q, q)),
                     (dict(frame_tokens=4), (q[..., :256], q[..., :256], q[..., :256])),
                     (dict(frame_tokens=4), (q, q, q[:, :4]))):
        with pytest.raises(fake_frames.OsbError):
            fake_frames.attn_frames(*args, **kw)
    assert fake_frames.launch_count() == 0


# ---- the host switch on a small VAE with a 512-wide mid block ----------------------------------------------------------
def _vae512(**kw):
    from opensora.registry import MODELS, build_module

    torch.manual_seed(21)
    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 512, 512), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4, **kw), MODELS, device_map="cpu")
    return m.to(torch.bfloat16)


def _count_sdpa(monkeypatch):
    import torch.nn.functional as F

    n, real = [0], F.scaled_dot_product_attention

    def counting(*a, **k):
        n[0] += 1
        return real(*a, **k)

    monkeypatch.setattr(F, "scaled_dot_product_attention", counting)
    return n


@pytest.mark.parametrize("tiled", [False, True])
def test_native_attention_matches_the_sdpa_path(fake_frames, monkeypatch, tiled):
    m = _vae512(sample_size=16, sample_tsize=64, use_spatial_tiling=tiled)
    sdpa = _count_sdpa(monkeypatch)
    torch.manual_seed(2)
    x = torch.rand(1, 3, 9, 32, 32) * 2 - 1          # 3 latent frames of 4 x 4 (tiled: tiles of 2 x 2 latent positions)
    z = torch.randn(1, 4, 3, 4, 4)
    with torch.no_grad():
        ze0, yd0 = m.encode(x, sample_posterior=False), m.decode(z)
        off_sdpa, off_frames = sdpa[0], sum(c[0] == "attn_frames" for c in fake_frames.calls)
        m.enable_native_attention()
        fake_frames.reset()
        sdpa[0] = 0
        ze1, yd1 = m.encode(x, sample_posterior=False), m.decode(z)
        on_sdpa, on_frames = sdpa[0], sum(c[0] == "attn_frames" for c in fake_frames.calls)
        m.disable_native_attention()
        ze2, yd2 = m.encode(x, sample_posterior=False), m.decode(z)
        # the floor: how far the SDPA path itself moves when its attention is computed in fp32 and rounded once
        import torch.nn.functional as F
        real = F.scaled_dot_product_attention
        monkeypatch.setattr(F, "scaled_dot_product_attention", lambda q, k, v: real(q.float(), k.float(), v.float()).to(q.dtype))
        ze3, yd3 = m.encode(x, sample_posterior=False), m.decode(z)
    assert ze1.shape == ze0.shape and yd1.shape == yd0.shape
    assert rel_l2(ze1, ze0) < max(VAE_BAR, 1.5 * rel_l2(ze3, ze0)) and rel_l2(yd1, yd0) < max(VAE_BAR, 1.5 * rel_l2(yd3, yd0))
    # T = 3 SDPA calls per mid block become one attn_frames launch
    assert off_frames == 0 and on_sdpa == 0 and off_sdpa == 3 * on_frames and on_frames >= 2
    hw = {c[1][4] for c in fake_frames.calls if c[0] == "attn_frames"}                  # frame_tokens = H * W of the (tile's) latent
    assert (max(hw) <= 4 if tiled else hw == {16}) and all(c[1][5] == 0 for c in fake_frames.calls if c[0] == "attn_frames")
    assert torch.equal(ze2, ze0) and torch.equal(yd2, yd0), "disable_native_attention() restores the default path's bits"


def test_native_attention_refuses_another_width(fake_frames):
    from opensora.registry import MODELS, build_module

    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4), MODELS, device_map="cpu")
    with pytest.raises(ValueError, match="32 wide"):
        m.enable_native_attention()
    assert not any(a.native for a in m._mid_attentions())


def _shard_worker(rank, world, port, ret):
    import sys

    import torch.distributed as dist

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        fake_osb200.attn_frames = FA.attn_frames
        m = _vae512()
        m.enable_native_attention()
        torch.manual_seed(3)
        z, x = torch.randn(1, 4, 5, 4, 4), torch.rand(1, 3, 17, 32, 32) * 2 - 1     # 5 latent frames: 3 + 2 over two ranks
        with torch.no_grad():
            m.disable_native_attention()
            sdpa_y, sdpa_z = m.decode(z), m.encode(x, sample_posterior=False)
            m.enable_native_attention()
            whole_y, whole_z = m.decode(z), m.encode(x, sample_posterior=False)
            m.enable_temporal_parallel(dist.group.WORLD)
            fake_osb200.reset()
            shard_y, shard_z = m.decode(z), m.encode(x, sample_posterior=False)
        frames = [c[1] for c in fake_osb200.calls if c[0] == "attn_frames"]
        # floor: the distance between the two bf16 attention paths on one rank (this model's 512-wide random layers
        # amplify a flipped bf16 rounding more than the 32-wide model of test_host_vae_cpu.py does)
        ret[rank] = dict(rel_y=rel_l2(shard_y, whole_y), rel_z=rel_l2(shard_z, whole_z), frames=frames,
                         floor_y=rel_l2(whole_y, sdpa_y), floor_z=rel_l2(whole_z, sdpa_z))
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(900)
def test_frame_sharded_native_attention_matches_one_rank():
    import torch.multiprocessing as mp

    port = 29500 + (os.getpid() + 7) % 2000
    ret = mp.Manager().dict()
    mp.spawn(_shard_worker, args=(2, port, ret), nprocs=2, join=True)
    for r in range(2):
        o = ret[r]
        assert o["rel_y"] < max(VAE_BAR, 1.5 * o["floor_y"]) and o["rel_z"] < max(VAE_BAR, 1.5 * o["floor_z"]), (r, dict(o))
        # local queries (3 or 2 frames of 16 tokens) against the gathered 5 frames, offset by the rank's first frame
        assert o["frames"] and all(f[1] == (3 - r) * 16 and f[2] == 5 * 16 and f[4] == 16 and f[5] == 3 * r for f in o["frames"]), (r, o["frames"])


def test_attn_frames_args_layout_matches_header():
    import ctypes
    import subprocess
    import tempfile

    import osb200

    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    names = [f[0] for f in osb200.AttnFramesArgs._fields_]
    fields = [("sizeof(osb_attn_frames_args)", ctypes.sizeof(osb200.AttnFramesArgs))] + [
        (f"offsetof(osb_attn_frames_args, {f})", getattr(osb200.AttnFramesArgs, f).offset) for f in names]
    with tempfile.TemporaryDirectory() as d:
        src = os.path.join(d, "probe.c")
        with open(src, "w") as f:
            f.write('#include <stdio.h>\n#include <stddef.h>\n#include "osb200.h"\nint main(){\n')
            for expr, _ in fields:
                f.write(f'printf("%zu\\n", (size_t)({expr}));\n')
            f.write("return 0;}\n")
        exe = os.path.join(d, "probe")
        subprocess.check_call(["gcc", "-I", os.path.join(root, "include"), src, "-o", exe])
        got = [int(v) for v in subprocess.check_output([exe]).split()]
    for (expr, mine), theirs in zip(fields, got):
        assert mine == theirs, (expr, mine, theirs)
    assert "osb_attn_frames" in osb200.EXPORTS
