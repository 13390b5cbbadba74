"""Multi-GPU check (run under torchrun, NCCL): the sequence-parallel STDiT3 forward (T-sharded tokens,
all-to-all transposition around temporal attention, exit all-gather) must reproduce the single-GPU
forward of the same model on the same inputs.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 \
        --master-port 29511 tests/sp_gpu_check.py
"""
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
    from tests.models import stdit3_inputs, stdit3_pair
    from tests.util import rel_l2

    ok = True
    for cfg_name, (B, T, H, W) in (("xs", (2, 8, 16, 16)), ("xs", (1, 16, 8, 16))):
        prod, oracle, cfg = stdit3_pair(cfg_name, device=torch.device("cuda", local))
        inp = stdit3_inputs(cfg, B, T, H, W, lens=[300, 40][:B], device="cuda")
        xm = torch.ones(B, T, dtype=torch.bool, device="cuda")
        xm[0, 1] = False
        for x_mask in (None, xm):
            for exchange in ("peer", "nccl"):
                with torch.no_grad():
                    single = prod(**inp, x_mask=x_mask)
                    prod.enable_sequence_parallel(dist.group.WORLD, exchange=exchange)
                    sp = prod(**inp, x_mask=x_mask)
                    sp2 = prod(**inp, x_mask=x_mask)    # a second step through the same exchange buffers / epochs
                    kind = prod.sp_exchange_kind
                    prod.enable_sequence_parallel(None)
                r = rel_l2(sp, single)
                same = torch.equal(sp, single) and torch.equal(sp2, single)
                print(f"[sp{world}] rank {rank} {cfg_name} B{B} {T}x{H}x{W} x_mask={x_mask is not None} exchange={exchange} "
                      f"({kind[:40]}): rel_l2 vs single-GPU = {r:.3e} bit_identical={same}", flush=True)
                ok &= r < 2e-3
    t = torch.tensor([1.0 if ok else 0.0], device="cuda")
    dist.all_reduce(t, op=dist.ReduceOp.MIN)
    dist.destroy_process_group()
    if t.item() != 1.0:
        sys.exit(1)
    if rank == 0:
        print("SP_CHECK_OK")


if __name__ == "__main__":
    main()
