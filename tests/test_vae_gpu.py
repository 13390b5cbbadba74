"""GPU parity of the causal-VAE path (through the C ABI) against the oracle restatement of the reference
(`oracle/vae_oracle.py`, pinned by reference-executed goldens) on identical bf16-rounded weights / inputs, and
against the committed reference goldens themselves (tests/golden/vae_blocks.npz)."""
import os

import numpy as np
import pytest
import torch

from tests.util import load_golden, report

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def osb():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import osb200

    osb200.init(0)
    return osb200


def _ndhwc(x):
    return x.permute(0, 2, 3, 4, 1).contiguous()


def _ncdhw(x):
    return x.permute(0, 4, 1, 2, 3).contiguous()


def _rand(*shape, seed=0, scale=1.0):
    g = torch.Generator(device="cuda").manual_seed(seed)
    return (torch.randn(*shape, generator=g, device="cuda") * scale).to(torch.bfloat16)


@pytest.mark.parametrize("C,groups,shape", [(128, 32, (2, 3, 10, 12)), (32, 8, (1, 5, 7, 9)), (512, 32, (1, 2, 6, 6))])
def test_group_stats(osb, C, groups, shape):
    nb, T, H, W = shape
    x = _rand(nb, T, H, W, C, seed=1) * 2 + 0.3
    st = osb.group_stats(x, groups, 1e-6)
    xf = x.float().view(nb, T * H * W, groups, C // groups)
    mean = xf.mean(dim=(1, 3))
    var = xf.var(dim=(1, 3), unbiased=False)
    torch.testing.assert_close(st[..., 0], mean, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(st[..., 1], torch.rsqrt(var + 1e-6), rtol=1e-4, atol=1e-5)


def test_group_stats_large_mean_small_std(osb):
    """|mean| >> std (mean 60, std 0.25 after bf16 rounding): E[x^2] - mean^2 in fp32 partials would lose the variance; the
    kernel's shifted sums must not (torch.nn.GroupNorm uses Welford)."""
    nb, T, H, W, C, groups = 1, 4, 24, 24, 64, 8
    g = torch.Generator(device="cuda").manual_seed(7)
    x = (60.0 + 0.25 * torch.randn(nb, T, H, W, C, generator=g, device="cuda")).to(torch.bfloat16)
    st = osb.group_stats(x, groups, 1e-6)
    xf = x.double().view(nb, T * H * W, groups, C // groups)
    mean = xf.mean(dim=(1, 3))
    var = xf.var(dim=(1, 3), unbiased=False)
    assert float(var.min()) > 0.01
    torch.testing.assert_close(st[..., 0].double(), mean, rtol=1e-5, atol=1e-4)
    torch.testing.assert_close(st[..., 1].double(), torch.rsqrt(var + 1e-6), rtol=2e-3, atol=0)


@pytest.mark.parametrize("up", [(1, 1, 1), (2, 2, 2), (1, 2, 2)])
def test_vae_prep(osb, up):
    from oracle import vae_oracle as V

    nb, T, H, W, C, groups = 1, 3, 5, 6, 64, 8
    x = _rand(nb, T, H, W, C, seed=2)
    gamma, beta = _rand(C, seed=3) * 0.2 + 1, _rand(C, seed=4) * 0.1
    st = osb.group_stats(x, groups, 1e-6)
    y = osb.vae_prep(x, stats=st, gamma=gamma, beta=beta, groups=groups, silu=True, up=up, pad=(2, 1, 1))
    ref = V.group_norm_silu(_ncdhw(x.float()), gamma.float(), beta.float(), groups)
    if up != (1, 1, 1):
        ref = V.upsample_causal3d(ref, up)
    ref = torch.nn.functional.pad(ref, (1, 1, 1, 1, 2, 0), mode="replicate")
    r, _ = report(f"vae_prep up{up}", _ncdhw(y), ref)
    assert r < 3e-3 and y.shape == _ndhwc(ref).shape


CONV_CASES = [
    # cin, cout, (T,H,W), stride
    (64, 128, (3, 10, 12), (1, 1, 1)),
    (128, 128, (5, 16, 40), (1, 1, 1)),
    (128, 64, (5, 16, 16), (1, 2, 2)),
    (64, 64, (5, 12, 20), (2, 2, 2)),
    (8, 128, (4, 9, 33), (1, 1, 1)),     # narrow mode (video conv_in: 3 channels padded to 8)
    (16, 64, (3, 8, 8), (1, 1, 1)),      # narrow mode (latent conv_in)
    (256, 256, (2, 6, 130), (1, 1, 1)),  # wide W: 128-wide boxes + a ragged tail
]


@pytest.mark.parametrize("cin,cout,thw,stride", CONV_CASES)
def test_causal_conv3d(osb, cin, cout, thw, stride):
    from opensora.models.hunyuan_vae.unet_causal_3d_blocks import CausalConv3d
    from oracle import vae_oracle as V

    T, H, W = thw
    real_cin = 3 if cin == 8 else cin
    m = CausalConv3d(real_cin, cout, 3, stride=stride)
    with torch.no_grad():
        m.conv.weight.copy_(torch.randn_like(m.conv.weight) * (27 * real_cin) ** -0.5)
        m.conv.bias.copy_(torch.randn_like(m.conv.bias) * 0.1)
    m = m.cuda().to(torch.bfloat16)
    x = _rand(2, T, H, W, cin, seed=5)
    if real_cin != cin:
        x[..., real_cin:] = 0
    y = m(x)
    ref = V.causal_conv3d(_ncdhw(x.float())[:, :real_cin], m.conv.weight.float(), m.conv.bias.float(), stride)
    r, _ = report(f"conv {cin}->{cout} {thw} s{stride}", _ncdhw(y), ref)
    assert y.shape == _ndhwc(ref).shape
    assert r < 2.5e-3


def test_conv3d_with_residual_and_norm(osb):
    from opensora.models.hunyuan_vae.unet_causal_3d_blocks import ResnetBlockCausal3D
    from oracle import vae_oracle as V

    for cin, cout in ((64, 64), (64, 128)):
        m = ResnetBlockCausal3D(in_channels=cin, out_channels=cout, groups=8)
        with torch.no_grad():
            for n, p in m.named_parameters():
                if "norm" in n and n.endswith("weight"):
                    p.copy_(1 + 0.2 * torch.randn_like(p))
                elif p.dim() == 1:
                    p.copy_(0.1 * torch.randn_like(p))
        m = m.cuda().to(torch.bfloat16)
        x = _rand(1, 4, 10, 14, cin, seed=6)
        y = m(x)
        W = {k: v.float() for k, v in m.state_dict().items()}
        ref = V.resnet_block(W, "", _ncdhw(x.float()), groups=8)
        r, _ = report(f"resnet {cin}->{cout}", _ncdhw(y), ref)
        assert r < 6e-3  # two convolutions + two GroupNorms, each rounding to bf16 once


def test_encoder_decoder_against_reference_goldens(osb):
    """The committed fixture was produced by the REFERENCE's own encoder/decoder (fp32); our bf16 path must
    reproduce it within bf16 tolerance."""
    from opensora.registry import MODELS, build_module

    G = load_golden("vae_blocks.npz")
    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4), MODELS, device_map="cpu")
    m.encoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("enc.")})
    m.decoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("dec.")})
    m = m.cuda().to(torch.bfloat16)
    from oracle import vae_oracle as V
    from tests.util import rel_l2

    down, up = V.stage_plan(4, 4, 8)
    # noise floor: the reference arithmetic itself (oracle restatement) run in bf16 on the same inputs / weights
    Wb = {k: v.cuda().to(torch.bfloat16) for k, v in G.items()}
    ze_bf = V.encoder({k[4:]: v for k, v in Wb.items() if k.startswith("enc.")}, Wb["enc_x"], groups=4, strides=down)
    yd_bf = V.decoder({k[4:]: v for k, v in Wb.items() if k.startswith("dec.")}, Wb["enc_y"][:, :4], groups=4, factors=up)
    fe, fd = rel_l2(ze_bf, G["enc_y"].cuda()), rel_l2(yd_bf, G["dec_y"].cuda())
    print(f"[parity] reference-in-bf16 noise floor: encoder {fe:.3e} decoder {fd:.3e}")
    xin = m._to_ndhwc(G["enc_x"].cuda().to(torch.bfloat16), cpad=8)
    z = m._to_ncdhw(m.encoder(xin))
    r, _ = report("encoder vs reference golden", z, G["enc_y"].cuda())
    assert z.shape == G["enc_y"].shape and r < 1.15 * fe   # measured 1.07e-2 against the reference-in-bf16 floor 1.27e-2
    y = m._to_ncdhw(m.decoder(m._to_ndhwc(G["enc_y"][:, :4].cuda().to(torch.bfloat16))))
    r, _ = report("decoder vs reference golden", y, G["dec_y"].cuda())
    assert y.shape == G["dec_y"].shape and r < fd          # measured 2.11e-2 against 3.04e-2


def test_autoencoder_roundtrip_api(osb):
    from opensora.registry import MODELS, build_module

    torch.manual_seed(0)
    m = build_module(dict(type="hunyuan_vae", block_out_channels=(32, 64, 64, 64), layers_per_block=1, norm_num_groups=8,
                          latent_channels=16), MODELS, device_map="cuda")
    x = torch.rand(1, 3, 9, 64, 64, device="cuda") * 2 - 1
    with torch.no_grad():
        z = m.encode(x, sample_posterior=False)
        assert list(z.shape) == [1, 16] + m.get_latent_size([9, 64, 64])
        x_rec, posterior, z2 = m(x, sample_posterior=False)
    assert x_rec.shape == x.shape and torch.isfinite(x_rec).all()
    d = float((z.float() - z2.float()).abs().max())
    print(f"[determinism] encode twice: max |z - z2| = {d:.3e}, identical={torch.equal(z, z2)}")
    assert d < 2e-2


def test_conv_causality_on_gpu(osb):
    """CausalConv3d (unet_causal_3d_blocks.py:63-96): perturbing the last frame leaves every earlier output frame
    bit-identical.  (The full VAE is NOT causal end to end - GroupNorm statistics span all frames, in the reference too.)"""
    from opensora.models.hunyuan_vae.unet_causal_3d_blocks import CausalConv3d

    m = CausalConv3d(64, 64, 3).cuda().to(torch.bfloat16)
    x = _rand(1, 6, 9, 11, 64, seed=9)
    y0 = m(x)
    x2 = x.clone()
    x2[:, -1] += 1.0
    y1 = m(x2)
    assert torch.equal(y0[:, :-1], y1[:, :-1]) and not torch.equal(y0[:, -1], y1[:, -1])


@pytest.mark.parametrize("tag,sp,tp", [("none", False, False), ("spatial", True, False), ("temporal", False, True), ("both", True, True)])
def test_tiled_modes_against_reference_goldens(osb, tag, sp, tp):
    """Tiled / blended encode + decode (autoencoder_kl_causal_3d.py:384-552) vs the reference class executed in fp32
    (tests/golden/vae_tiled.npz); tolerance = the reference arithmetic itself in bf16 (noise floor) x 1.5."""
    from opensora.registry import MODELS, build_module
    from oracle import vae_oracle as V
    from tests.util import rel_l2

    G = load_golden("vae_blocks.npz")
    GT = load_golden("vae_tiled.npz")
    m = build_module(dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4,
                          latent_channels=4, sample_size=32, sample_tsize=8, use_spatial_tiling=sp, use_temporal_tiling=tp),
                     MODELS, device_map="cpu")
    m.encoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("enc.")})
    m.decoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("dec.")})
    with torch.no_grad():
        m.quant_conv.weight.copy_(GT["quant_w"]); m.quant_conv.bias.copy_(GT["quant_b"])
        m.post_quant_conv.weight.copy_(GT["post_w"]); m.post_quant_conv.bias.copy_(GT["post_b"])
    m = m.cuda().to(torch.bfloat16)
    with torch.no_grad():
        z = m.encode(GT["x"].cuda(), sample_posterior=False)
        y = m.decode(GT[f"z_{tag}"].cuda())
    # noise floor: oracle (restated reference) in bf16
    down, up = V.stage_plan(4, 4, 8)
    bf = lambda d, pfx: {k[len(pfx):]: v.cuda().to(torch.bfloat16) for k, v in d.items() if k.startswith(pfx)}  # noqa: E731
    We, Wd = bf(G, "enc."), bf(G, "dec.")
    qw, qb, pw, pb = (GT[k].cuda().to(torch.bfloat16) for k in ("quant_w", "quant_b", "post_w", "post_b"))
    encode, decode = V.tiled_autoencoder(lambda x: V.causal_conv3d(V.encoder(We, x, groups=4, strides=down), qw, qb),
                                         lambda t: V.decoder(Wd, V.causal_conv3d(t, pw, pb), groups=4, factors=up),
                                         sample_size=32, sample_tsize=8, spatial=sp, temporal=tp)
    zf = rel_l2(0.476986 * encode(GT["x"].cuda().to(torch.bfloat16))[:, :4], GT[f"z_{tag}"].cuda())
    yf = rel_l2(decode((GT[f"z_{tag}"].cuda() / 0.476986).to(torch.bfloat16)), GT[f"y_{tag}"].cuda())
    rz, _ = report(f"tiled encode [{tag}]", z, GT[f"z_{tag}"].cuda())
    ry, _ = report(f"tiled decode [{tag}]", y, GT[f"y_{tag}"].cuda())
    print(f"[parity] reference-in-bf16 noise floor: encode {zf:.3e} decode {yf:.3e}")
    assert z.shape == GT[f"z_{tag}"].shape and y.shape == GT[f"y_{tag}"].shape
    assert rz < 1.1 * zf and ry < yf
