"""Multi-GPU check (run under torchrun, NCCL): the MMDiT drop-in with the joint txt|img sequence split over the ranks
(`MMDiTModel.enable_sequence_parallel`: Ulysses heads<->sequence all-to-all around every attention, var-len exit gather)
against the same model's single-GPU forward on the real kernels.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29514 tests/mmdit_sp_gpu_check.py

NOT yet run on a GPU box (written after the round's GPU budget was spent); CPU twin on gloo ranks:
tests/test_host_mmdit_cpu.py::test_mmdit_ulysses_sequence_parallel_world2 (bit-identical)."""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "open-sora_b200"))
import torch
import torch.distributed as dist


def main():
    rank, world = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"])
    local = int(os.environ.get("LOCAL_RANK", rank))
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    from tests.models import mmdit_ids, mmdit_model
    from tests.util import rel_l2

    ok = True
    for fused, liger, (B, Lt, T, H, W) in ((True, False, (2, 40, 3, 6, 8)), (False, True, (1, 64, 5, 12, 16))):
        m = mmdit_model(fused, liger, device="cuda")          # seeded: the same model on every rank; num_heads = 2 -> world 2 only
        if m.config.num_heads % world:
            if rank == 0:
                print(f"[mmdit-sp{world}] {m.config.num_heads} heads do not divide over {world} ranks: skipped")
            continue
        g = torch.Generator().manual_seed(3)
        rb = lambda *s: torch.randn(*s, generator=g).to(torch.bfloat16)  # noqa: E731
        txt_ids, img_ids = mmdit_ids(B, Lt, T, H, W)
        inp = dict(img=rb(B, T * H * W, 64), img_ids=img_ids, txt=rb(B, Lt, 128), txt_ids=txt_ids, timesteps=torch.rand(B, generator=g),
                   y_vec=rb(B, 96), cond=rb(B, T * H * W, 68), guidance=torch.full((B,), 4.0))
        inp = {k: v.cuda() for k, v in inp.items()}
        with torch.no_grad():
            single = m(**inp)
            m.enable_sequence_parallel(dist.group.WORLD)
            sharded = m(**inp)
            again = m(**inp)
            m.enable_sequence_parallel(None)
        r = rel_l2(sharded, single)
        print(f"[mmdit-sp{world}] rank {rank} fused_qkv={fused} liger={liger} L={Lt + T * H * W}: rel_l2 vs single GPU = {r:.3e} "
              f"bit_identical={torch.equal(sharded, single)} repeatable={torch.equal(sharded, again)}", flush=True)
        ok &= sharded.shape == single.shape and r < 5e-3
    t = torch.tensor([1.0 if ok else 0.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    if t.item() != 1.0:
        sys.exit(1)
    if rank == 0:
        print("MMDIT_SP_CHECK_OK")


if __name__ == "__main__":
    main()
