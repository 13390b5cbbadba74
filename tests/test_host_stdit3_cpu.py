"""Host-side logic of the STDiT3 drop-in on the CPU: the real `opensora.models.stdit.stdit3.STDiT3` forward driven
through the CPU stand-in of the binding (tests/fake_osb200.py) and compared with the fp32 oracle.  What this pins
without a GPU: patch embedding and un-patchify permutes, the per-step modulation table and its `x_mask` index, the
packed kv projection of all blocks, the row-stride conventions handed to spatial / temporal / cross attention, ragged
text masks, and the sequence-parallel T-shard <-> S-shard transposition (gloo, world size 2) on the real model."""
import os

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from tests.models import stdit3_inputs, stdit3_pair
from tests.util import rel_l2


@pytest.mark.parametrize("B,T,H,W", [(1, 4, 8, 8), (2, 3, 6, 10)])
def test_forward_matches_oracle(fake_osb, B, T, H, W):
    prod, oracle, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, B, T, H, W)
    with torch.no_grad():
        ref = oracle(**inp)
        out = prod(**inp)
        noise = oracle.to(torch.bfloat16)(**inp).float()
    assert out.shape == ref.shape and out.dtype == torch.float32
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    assert r < max(1.5 * rn, 4e-3), (r, rn)
    # the boundary was driven as designed: every Linear is a gemm call, 3 attention calls and 2 LN calls per block + final LN
    names = [c[0] for c in fake_osb.calls]
    nb = 2 * cfg.depth
    assert names.count("attn_tiles") == 2 * nb and names.count("attn_short") == 0
    assert names.count("ln_modulate") == 2 * nb + 1
    kv = [c for c in fake_osb.calls if c[0] == "gemm" and c[1][1] == nb * 2 * cfg.hidden_size]
    assert len(kv) == 1, "all blocks' kv_linear run as ONE GEMM"


def test_x_mask_and_ragged_text(fake_osb):
    prod, oracle, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, 2, 4, 8, 8, lens=[cfg.model_max_length, 7])
    xm = torch.ones(2, 4, dtype=torch.bool)
    xm[0, 1:] = False
    xm[1, 0] = False
    with torch.no_grad():
        ref = oracle(**inp, x_mask=xm)
        out = prod(**inp, x_mask=xm)
        noise = oracle.to(torch.bfloat16)(**inp, x_mask=xm).float()
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    assert r < max(1.5 * rn, 4e-3), (r, rn)


def test_non_multiple_sizes_are_padded_and_cropped(fake_osb):
    prod, oracle, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, 1, 3, 7, 9)      # H, W not multiples of the (1,2,2) patch
    with torch.no_grad():
        ref = oracle(**inp)
        out = prod(**inp)
    assert out.shape == ref.shape == inp["x"].shape[:1] + (ref.shape[1],) + inp["x"].shape[2:]
    assert rel_l2(out, ref) < 2e-2


def test_dtype_contract_is_enforced(fake_osb):
    prod, _, cfg = stdit3_pair("xs", device="cpu")
    with pytest.raises(fake_osb.OsbError):
        prod.float()(**stdit3_inputs(cfg, 1, 2, 4, 4))


def _sp_worker(rank, world, port, ret):
    import sys

    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    try:
        from tests import fake_osb200

        sys.modules["osb200"] = fake_osb200
        torch.manual_seed(0)
        prod, _, cfg = stdit3_pair("xs", device="cpu")
        inp = stdit3_inputs(cfg, 2, 4, 8, 8, lens=[cfg.model_max_length, 9])
        xm = torch.ones(2, 4, dtype=torch.bool)
        xm[1, 2:] = False
        with torch.no_grad():
            single = prod(**inp, x_mask=xm)
            prod.enable_sequence_parallel(dist.group.WORLD)
            sharded = prod(**inp, x_mask=xm)
            # the reference's own switch: config flag + opensora.acceleration.parallel_states registry
            from opensora.acceleration.parallel_states import set_sequence_parallel_group

            prod.enable_sequence_parallel(None)
            prod.config.enable_sequence_parallelism = True
            set_sequence_parallel_group(dist.group.WORLD)
            via_config = prod(**inp, x_mask=xm)
        ret[rank] = bool(torch.equal(single, sharded)) and bool(torch.equal(single, via_config)) and prod._sp_group is not None
    finally:
        dist.destroy_process_group()


@pytest.mark.timeout(300)
def test_sequence_parallel_model_world2_is_bit_identical():
    """The real model, T-sharded over two gloo ranks with the all-to-all around every temporal attention, reproduces the
    single-rank output bit for bit (token-local ops do not care about the shard; attention sees whole sequences)."""
    port = 29500 + (os.getpid() + 7) % 2000
    mgr = mp.Manager()
    ret = mgr.dict()
    mp.spawn(_sp_worker, args=(2, port, ret), nprocs=2, join=True)
    assert ret.get(0) is True and ret.get(1) is True


def test_rflow_sampler_drives_the_model(fake_osb):
    """The v1.2 sampling loop (`opensora/schedulers/rf.py`: CFG batch of 2 with the model's own null caption, velocity half of
    the `pred_sigma` output, fused combine + Euler update) around the REAL host-side STDiT3, against the oracle loop around the
    fp32 oracle model: three steps, ragged caption mask."""
    from opensora.schedulers import RFLOW
    from oracle import sampling_oracle as S

    prod, oracle, cfg = stdit3_pair("xs", device="cpu")
    inp = stdit3_inputs(cfg, 2, 4, 8, 8, lens=[cfg.model_max_length, 11])
    B = 2
    y_null = prod.y_embedder.y_embedding.detach()[None, None].repeat(B, 1, 1, 1)
    extra = dict(fps=inp["fps"], height=inp["height"], width=inp["width"])
    z0 = inp["x"].to(torch.bfloat16)
    with torch.no_grad():
        ref = S.rflow_sample(lambda x, t, y, **kw: oracle(x, t, y, **kw), z0.float(), inp["y"], y_null.float(), mask=inp["mask"],
                             steps=3, cfg_scale=4.0, **extra)
        out = RFLOW(num_sampling_steps=3, cfg_scale=4.0).sample(prod, z0, inp["y"], y_null, mask=inp["mask"], additional_args=extra)
        # the reference-precision floor of the same loop: the oracle model in bf16, latent rounded to bf16 after every step
        ob = oracle.to(torch.bfloat16)
        noise = S.rflow_sample(lambda x, t, y, **kw: ob(x.to(torch.bfloat16).float(), t, y, **kw).float(), z0.float(), inp["y"],
                               y_null.float(), mask=inp["mask"], steps=3, cfg_scale=4.0, **extra)
    assert out.shape == z0.shape and out.dtype == torch.bfloat16
    r, rn = rel_l2(out, ref), rel_l2(noise, ref)
    # guidance amplifies the model's bf16 error (v = v_u + 4 (v_c - v_u)); a wrong branch order / sign / dt would be O(1)
    assert r < max(1.5 * rn, 1e-2) and r < 6e-2, (r, rn)
    assert [c[0] for c in fake_osb.calls].count("cfg_euler") == 3
