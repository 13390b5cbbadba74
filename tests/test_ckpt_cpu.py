"""`opensora/utils/ckpt.py` (inference-side mirror of the reference module, SURVEY.md 8f-4 "safetensors loading path"):
the three checkpoint kinds, key renaming, strictness, the offline hub-cache lookup, and the model factories loading through
it with the reference's state-dict keys."""
import json
import logging
import os

import pytest
import torch

from tests.util import load_golden
import torch.nn as nn
from safetensors.torch import save_file


class _Toy(nn.Module):
    def __init__(self):
        super().__init__()
        self.a = nn.Linear(4, 3)
        self.blocks = nn.ModuleList([nn.Linear(3, 3) for _ in range(2)])


def _sd(seed=0):
    torch.manual_seed(seed)
    return {k: torch.randn_like(v) for k, v in _Toy().state_dict().items()}


def _same(m, sd):
    return all(torch.equal(v, sd[k]) for k, v in m.state_dict().items())


def test_safetensors_pt_and_sharded_directory(tmp_path):
    from opensora.utils.ckpt import load_checkpoint

    sd = _sd()
    save_file(sd, str(tmp_path / "w.safetensors"))
    torch.save(sd, str(tmp_path / "w.pt"))
    assert _same(load_checkpoint(_Toy(), str(tmp_path / "w.safetensors")), sd)
    assert _same(load_checkpoint(_Toy(), str(tmp_path / "w.pt")), sd)
    # sharded: <dir>/model/{shards, index json with a weight_map}
    root = tmp_path / "epoch0" / "model"
    root.mkdir(parents=True)
    keys = sorted(sd)
    parts = {"model-00001.safetensors": keys[:3], "model-00002.safetensors": keys[3:]}
    for name, ks in parts.items():
        save_file({k: sd[k] for k in ks}, str(root / name))
    (root / "model.safetensors.index.json").write_text(json.dumps({"weight_map": {k: n for n, ks in parts.items() for k in ks}}))
    assert _same(load_checkpoint(_Toy(), str(tmp_path / "epoch0")), sd)
    (tmp_path / "weights.unknown").write_text("")
    with pytest.raises(ValueError, match="Invalid checkpoint path"):   # neither a known file kind nor a directory
        load_checkpoint(_Toy(), str(tmp_path / "weights.unknown"))


def test_rename_keys_strict_and_warnings(tmp_path, caplog):
    from opensora.utils.ckpt import load_checkpoint

    sd = _sd(1)
    old = {k.replace("blocks.", "layers."): v for k, v in sd.items()}
    save_file(old, str(tmp_path / "old.safetensors"))
    assert _same(load_checkpoint(_Toy(), str(tmp_path / "old.safetensors"), rename_keys={"layers.": "blocks."}), sd)
    with caplog.at_level(logging.WARNING, logger="opensora"):
        m = load_checkpoint(_Toy(), str(tmp_path / "old.safetensors"))       # strict=False: reported, not fatal
    assert "4 missing keys" in caplog.text and "4 unexpected keys" in caplog.text and "layers.0.weight" in caplog.text
    assert torch.equal(m.a.weight, sd["a.weight"])
    with pytest.raises(RuntimeError):
        load_checkpoint(_Toy(), str(tmp_path / "old.safetensors"), strict=True)


def test_hub_path_resolves_from_the_local_cache_only(tmp_path):
    from opensora.utils.ckpt import load_checkpoint, load_from_hf_hub

    sd = _sd(2)
    snap = tmp_path / "models--hpcai-tech--Open-Sora-v2" / "snapshots" / "abc123"
    snap.mkdir(parents=True)
    save_file(sd, str(snap / "Open_Sora_v2.safetensors"))
    assert load_from_hf_hub("hpcai-tech/Open-Sora-v2/Open_Sora_v2.safetensors", str(tmp_path)).startswith(str(snap))
    assert _same(load_checkpoint(_Toy(), "hpcai-tech/Open-Sora-v2/Open_Sora_v2.safetensors", cache_dir=str(tmp_path)), sd)
    with pytest.raises(FileNotFoundError, match="no network"):
        load_checkpoint(_Toy(), "hpcai-tech/Open-Sora-v2/absent.safetensors", cache_dir=str(tmp_path))


def test_model_factories_load_reference_keyed_checkpoints(tmp_path):
    """A checkpoint written with the reference's state-dict keys (here: the golden VAE weights produced by the executed
    reference classes, and an MMDiT state dict in the reference's un-fused qkv layout) loads through the factories."""
    import numpy as np

    from opensora.registry import MODELS, build_module
    from tests.models import MMDIT_CFG

    G = load_golden("vae_blocks.npz")
    kw = dict(type="hunyuan_vae", block_out_channels=(16, 32, 32, 32), layers_per_block=1, norm_num_groups=4, latent_channels=4)
    src = build_module(dict(kw), MODELS, device_map="cpu")
    src.encoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("enc.")})
    src.decoder.load_state_dict({k[4:]: v for k, v in G.items() if k.startswith("dec.")})
    save_file({k: v.contiguous() for k, v in src.state_dict().items()}, str(tmp_path / "vae.safetensors"))
    vae = build_module(dict(kw, from_pretrained=str(tmp_path / "vae.safetensors")), MODELS, device_map="cpu")
    assert all(torch.equal(v.float(), src.state_dict()[k].to(torch.bfloat16).float()) for k, v in vae.state_dict().items())
    bad = {k: v.contiguous() for k, v in src.state_dict().items() if "conv_in" not in k}
    save_file(bad, str(tmp_path / "vae_bad.safetensors"))
    with pytest.raises(RuntimeError):   # the VAE factory loads strictly (autoencoder_kl_causal_3d.py:636)
        build_module(dict(kw, from_pretrained=str(tmp_path / "vae_bad.safetensors")), MODELS, device_map="cpu")

    flux = build_module(dict(type="flux", **MMDIT_CFG), MODELS, device_map="cpu", torch_dtype=torch.float32)
    sd = {k: torch.randn_like(v) for k, v in flux.state_dict().items()}
    save_file(sd, str(tmp_path / "flux.safetensors"))
    again = build_module(dict(type="flux", from_pretrained=str(tmp_path / "flux.safetensors"), **MMDIT_CFG), MODELS, device_map="cpu",
                         torch_dtype=torch.float32)
    assert all(torch.equal(v, sd[k]) for k, v in again.state_dict().items())
