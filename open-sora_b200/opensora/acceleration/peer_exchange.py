"""Peer-memory exchange for sequence parallelism: the osb200 replacement of the reference's autograd all_to_all
(`opensora/acceleration/communications.py:8-18,57-63`) on the STDiT3 path.

The reference packs, calls `dist.all_to_all`, and unpacks around every temporal attention.  Here the kernels that
PRODUCE the data (LayerNorm+modulate before the temporal QKV projection, the attention kernel's epilogue after it) store
each row directly into the buffer of the rank that consumes it, through peer-mapped symmetric memory
(`torch.distributed._symmetric_memory`, NVLink 5 / NVSwitch), and one tiny barrier kernel (`osb_comm_barrier`) orders
producers and consumers across ranks.  No pack copy, no collective call, no unpack copy; everything is CUDA-graph
capturable.  PyTorch only allocates / maps the memory - NCCL is not on this path.

Buffer reuse is safe without double buffering: a rank can only reach exchange k+1 after it received every peer's data
of exchange k(b), which each peer sends after it finished reading exchange k(a) (see DESIGN.md 6)."""
from __future__ import annotations

import torch
import torch.distributed as dist


def scatter_dest(mode: int, P: int, rank: int, I: int, J: int, row: int) -> tuple[int, int]:
    """Host mirror of the device routing (`scatter_row`, open-sora_b200/csrc/common.cuh; include/osb200.h `osb_scatter`):
    row `row` of a [B, I, J] producer on `rank` -> (destination rank, row in its buffer).  mode 1 splits J
    ([B, Tl, S] -> [B, T, S/P]), mode 2 splits I ([B, T, Sl] -> [B, T/P, S]), mode 3 transposes locally
    ([B, T, S] -> [B, S, T]), mode 4 = mode 1 with the destination transposed ([B, Tl, S] -> [B, S/P, T])."""
    b, rem = divmod(row, I * J)
    i, j = divmod(rem, J)
    if mode == 1:
        jc = J // P
        p = j // jc
        return p, (b * P * I + rank * I + i) * jc + (j - p * jc)
    if mode == 3:
        return rank, (b * J + j) * I + i
    if mode == 4:
        jc = J // P
        p = j // jc
        return p, (b * jc + (j - p * jc)) * (P * I) + rank * I + i
    ic = I // P
    p = i // ic
    return p, (b * ic + (i - p * ic)) * (P * J) + rank * J + j


class PeerExchange:
    def __init__(self, group, device):
        import torch.distributed._symmetric_memory as symm

        import osb200

        self._symm, self._osb = symm, osb200
        self.group, self.device = group, device
        self.P, self.rank = dist.get_world_size(group), dist.get_rank(group)
        if self.P > osb200.MAX_PEERS:
            raise RuntimeError(f"peer exchange supports up to {osb200.MAX_PEERS} ranks, got {self.P}")
        self.group_name = group.group_name if hasattr(group, "group_name") else dist.group.WORLD.group_name
        enable = getattr(symm, "enable_symm_mem_for_group", None)
        if enable is not None:
            try:
                enable(self.group_name)
            except Exception:
                pass   # newer torch: implicit
        import os

        self._debug_sync = os.environ.get("OSB_SP_DEBUG_SYNC", "0") == "1"
        self._bufs: dict = {}
        flags, self._flag_ptrs = self._alloc((64,), torch.int32)
        flags.zero_()
        self.flags = flags
        self.epoch = torch.zeros(1, dtype=torch.int32, device=device)
        torch.cuda.synchronize(device)
        dist.barrier(group)   # every rank's flags are zero before anyone signals

    def _alloc(self, shape, dtype):
        t = self._symm.empty(*shape, dtype=dtype, device=self.device)
        hdl = self._symm.rendezvous(t, self.group_name)
        return t, [int(p) for p in hdl.buffer_ptrs]

    def buffer(self, key, rows: int, cols: int):
        """Symmetric bf16 [rows, cols] receive buffer (allocated collectively on first use, then cached)."""
        k = (key, rows, cols)
        if k not in self._bufs:
            self._bufs[k] = self._alloc((rows, cols), torch.bfloat16)
        return self._bufs[k]

    def scatter(self, mode: int, I: int, J: int, peer_ptrs):
        return self._osb.make_scatter(mode, self.P, self.rank, I, J, peer_ptrs)

    def barrier(self) -> None:
        if self._debug_sync:   # OSB_SP_DEBUG_SYNC=1: host-side barrier instead of the flag kernel (debugging aid)
            torch.cuda.synchronize(self.device)
            dist.barrier(self.group)
            return
        self._osb.comm_barrier(self.P, self.rank, self.epoch, self._flag_ptrs[self.rank], self._flag_ptrs)
