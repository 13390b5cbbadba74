"""osb_attn_frames on the GPU, through the C ABI (the frame-causal attention of one 512-wide head that
`AutoencoderKLCausal3D.enable_native_attention()` switches the VAE's mid block to): the kernel against an fp32 torch
restatement with an explicit mask on identical bf16 inputs, causality and determinism as bit-level properties, the CPU
tests' stand-in against the kernel, the refusals, and a small VAE with a 512-wide mid block against its SDPA path and
against the fp32 oracle."""
import pytest
import torch

from tests import fake_osb200 as F_
from tests.util import rel_l2, report

pytestmark = pytest.mark.gpu
BAR = 4e-3   # the bf16 attention bar of the other attention kernels


@pytest.fixture(scope="module")
def osb():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import osb200

    osb200.init(0)
    return osb200


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


def restatement(q, k, v, hw, q_frame0=0, chunk=2048):
    """fp32 softmax(q k^T / sqrt(D) + mask) v with the mask of prepare_causal_attention_mask spelled out, in query
    chunks so that the 17 408-token shape fits."""
    Lq, Lk = q.shape[1], k.shape[1]
    kf, vf = k.float(), v.float()
    keys = torch.arange(Lk, device=q.device)
    out = []
    for i0 in range(0, Lq, chunk):
        i = torch.arange(i0, min(i0 + chunk, Lq), device=q.device)
        s = q[:, i0:i0 + chunk].float() @ kf.transpose(1, 2) * q.shape[-1] ** -0.5
        dead = keys[None, :] >= torch.clamp((q_frame0 + i // hw + 1) * hw, max=Lk)[:, None]
        out.append(torch.softmax(s.masked_fill(dead[None], float("-inf")), -1) @ vf)
    return torch.cat(out, 1)


@pytest.mark.parametrize("hw,T,extra", [(64, 3, 0), (128, 2, 0), (4, 40, 0), (100, 5, 0), (1000, 3, 0), (64, 1, 0),
                                        (50, 3, -13), (1024, 17, 0)])
def test_kernel_matches_the_fp32_restatement(osb, hw, T, extra):
    """Aligned frames (64, 128), 16 frames inside one query tile (4), frames that straddle tiles and key blocks (100,
    1000), one frame, a length that is no multiple of 64 or of the frame, and the reference's tile: 17 x 32 x 32."""
    L = T * hw + extra
    q, k, v = (_rand(1, L, 512, seed=s + hw) for s in range(3))
    out = osb.attn_frames(q, k, v, frame_tokens=hw)
    torch.cuda.synchronize()
    assert report(f"attn_frames hw {hw} L {L}", out, restatement(q, k, v, hw))[0] < BAR


def test_batch_column_slices_and_frame_offset(osb):
    """Two samples with batch strides, q | k | v as column slices of one [rows, 1536] buffer, local queries of frames 2, 3
    against the keys of 5 frames (frame-sharded VAE), out into a strided buffer."""
    hw, Tq, Tk, first = 72, 2, 5, 2
    buf = _rand(2, Tk * hw + 7, 1536, seed=9)
    q, k, v = buf[:, first * hw:(first + Tq) * hw, :512], buf[:, :Tk * hw, 512:1024], buf[:, :Tk * hw, 1024:]
    obuf = torch.full((2, Tk * hw + 7, 640), 7.0, device="cuda", dtype=torch.bfloat16)   # out has q's batch stride in rows
    out = osb.attn_frames(q, k, v, frame_tokens=hw, q_frame0=first, out=obuf[:, first * hw:(first + Tq) * hw, :512])
    torch.cuda.synchronize()
    assert report("attn_frames sliced", out, restatement(q, k, v, hw, first))[0] < BAR
    assert bool((obuf[:, :first * hw] == 7).all()) and bool((obuf[:, (first + Tq) * hw:] == 7).all()) and \
        bool((obuf[..., 512:] == 7).all()), "nothing outside out is written"


def test_causality_determinism_and_range(osb):
    hw, T = 200, 4
    q, k, v = (_rand(1, T * hw, 512, seed=20 + s) for s in range(3))
    out = osb.attn_frames(q, k, v, frame_tokens=hw)
    again = osb.attn_frames(q, k, v, frame_tokens=hw)
    k2, v2 = k.clone(), v.clone()
    k2[:, -hw:] = _rand(1, hw, 512, seed=30) * 3
    v2[:, -hw:] = _rand(1, hw, 512, seed=31) * 3
    out2 = osb.attn_frames(q, k2, v2, frame_tokens=hw)
    torch.cuda.synchronize()
    assert torch.equal(out, again), "a second call gives the same bits"
    assert torch.equal(out2[:, :-hw], out[:, :-hw]), "the last frame's keys / values reach no earlier frame"
    assert not torch.equal(out2[:, -hw:], out[:, -hw:])
    big = osb.attn_frames(q * 30, k * 30, v, frame_tokens=hw)       # scores ~ 900x: one key dominates each row
    torch.cuda.synchronize()
    assert bool(torch.isfinite(big).all())
    assert report("attn_frames x30", big, restatement(q * 30, k * 30, v, hw))[0] < BAR


def test_stand_in_matches_the_kernel(osb):
    """Pins the stand-in's attn_frames (tests/fake_osb200.py), which the CPU tests of the host switch rely on."""
    hw, Tq, Tk, first = 36, 3, 6, 1
    q, k, v = _rand(2, Tq * hw, 512, seed=40), _rand(2, Tk * hw, 512, seed=41), _rand(2, Tk * hw, 512, seed=42)
    out = osb.attn_frames(q, k, v, frame_tokens=hw, q_frame0=first)
    torch.cuda.synchronize()
    assert report("kernel vs stand-in", out, F_.attn_frames(q, k, v, frame_tokens=hw, q_frame0=first))[0] < BAR


def test_refusals_do_not_launch(osb):
    q = _rand(1, 128, 512, seed=50)
    n0 = osb.launch_count()
    wide = _rand(1, 128, 1024, seed=51)
    for args, kw, what in (((wide, wide, wide), dict(frame_tokens=64), "head_dim"),
                           ((q[..., :256],) * 3, dict(frame_tokens=64), "head_dim"),
                           ((q, q, q), dict(frame_tokens=0), "frame_tokens"),
                           ((q, q, q), dict(frame_tokens=64, q_frame0=-1), "no key")):
        with pytest.raises(osb.OsbError, match=what):
            osb.attn_frames(*args, **kw)
    # a leading dimension below 512 cannot be expressed through the binding's tensors: straight through the C ABI
    import ctypes as C

    a = osb.AttnFramesArgs()
    a.q = a.k = a.v = a.out = q.data_ptr()
    a.q_ld, a.k_ld, a.v_ld, a.out_ld = 512, 256, 512, 512
    a.q_batch_stride = a.k_batch_stride = a.Lq = a.Lk = 128
    a.batch, a.head_dim, a.frame_tokens, a.q_frame0, a.softmax_scale = 1, 512, 64, 0, 512 ** -0.5
    assert osb._lib.osb_attn_frames(C.byref(a), None) != 0 and "leading dimensions" in osb.last_error()
    torch.cuda.synchronize()
    assert osb.launch_count() == n0


def test_vae_with_native_attention(osb):
    """A small VAE whose mid block is 512 wide: native attention against the SDPA path and against the fp32 oracle; the
    bar is the distance of the oracle run in bf16 from the oracle in fp32, as in test_vae_gpu.py."""
    from opensora.registry import MODELS, build_module
    from oracle import vae_oracle as V

    torch.manual_seed(21)
    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 512, 512), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4), MODELS, device_map="cuda").eval()
    x = (torch.rand(1, 3, 9, 64, 64, device="cuda") * 2 - 1).to(torch.bfloat16)      # 3 latent frames of 8 x 8
    z = torch.randn(1, 4, 3, 8, 8, device="cuda").to(torch.bfloat16)
    down, up = V.stage_plan(4, 4, 8)
    sd = lambda mod, dt: {k: v.detach().to(dt) for k, v in mod.state_dict().items()}  # noqa: E731  (bf16 parameters)
    with torch.no_grad():
        lat_ref = V.encoder(sd(m.encoder, torch.float32), x.float(), groups=4, strides=down)
        vid_ref = V.decoder(sd(m.decoder, torch.float32), z.float(), groups=4, factors=up)
        lat_bf = V.encoder(sd(m.encoder, torch.bfloat16), x, groups=4, strides=down)
        vid_bf = V.decoder(sd(m.decoder, torch.bfloat16), z, groups=4, factors=up)
        enc = lambda: m._to_ncdhw(m.encoder(m._to_ndhwc(x, cpad=8)))   # noqa: E731
        dec = lambda: m._to_ncdhw(m.decoder(m._to_ndhwc(z)))          # noqa: E731
        lat0, vid0 = enc(), dec()
        m.enable_native_attention()
        n0 = osb.launch_count()
        lat1, vid1 = enc(), dec()
        torch.cuda.synchronize()
    fl, fv = rel_l2(lat_bf, lat_ref), rel_l2(vid_bf, vid_ref)
    print(f"[parity] bf16 floor: latent {fl:.3e} video {fv:.3e}; launches with native attention {osb.launch_count() - n0}")
    assert report("native vs sdpa latent", lat1, lat0)[0] < max(1.5 * fl, 1e-2)
    assert report("native vs sdpa video", vid1, vid0)[0] < max(1.5 * fv, 1e-2)
    assert report("native vs oracle latent", lat1, lat_ref)[0] < max(1.5 * fl, 1e-2)
    assert report("native vs oracle video", vid1, vid_ref)[0] < max(1.5 * fv, 1e-2)
