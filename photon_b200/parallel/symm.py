"""Symmetric device memory over NVLink: one arena per rank, mapped into every peer.

The fused round kernels (R1/R2) and the DDP all-reduce (N1) address *peer*
memory directly (P2P loads/stores through NVSwitch), so every rank allocates the
same set of named planes at the same offsets and exchanges CUDA IPC handles
once (bootstrap only — no NCCL call ever touches the planes).  Two modes:

* ``distributed``: one process per GPU (``torchrun``); handles travel through
  ``torch.distributed.all_gather_object``;
* ``single``: one process driving several local GPUs with peer access enabled
  (unit tests, notebooks).

When the box exposes NVLink SHARP (NVLS) the distributed arena is allocated through
``torch.distributed._symmetric_memory`` instead of CUDA IPC: besides the per-peer pointers it then
has a MULTICAST mapping (``mc_ptr``) on which the kernels use ``multimem.ld_reduce`` (the sum over
all GPUs is formed inside the NVSwitch) and ``multimem.st`` (one store reaches every GPU).
``PB_NVLS=0`` forces the IPC / P2P path.

Replaces the reference's host-side hand-off stack (POSIX shm / Ray plasma / S3;
ref: photon/server/s3_utils.py:730-1115, photon/shm/utils.py) on the GPU path.
"""
from __future__ import annotations

from typing import Any

import os

import torch
import torch.distributed as dist

from photon_b200 import ops

_DT = {torch.float32: ("float32", 4), torch.bfloat16: ("bfloat16", 2), torch.float64: ("float64", 8), torch.int32: ("int32", 4),
       torch.uint8: ("uint8", 1)}
_ALIGN = 4096


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


class SymmArena:
    def __init__(self, planes: dict[str, tuple[int, torch.dtype]], *, rank: int = 0, world_size: int = 1,
                 device: torch.device | int | None = None, group: Any = None, devices: list[int] | None = None) -> None:
        """``planes``: name → (numel, dtype). ``devices`` selects single-process multi-GPU mode."""
        self.ext = ops.ext()
        self.single = devices is not None
        self.world_size = len(devices) if self.single else int(world_size)
        if not 1 <= self.world_size <= 8:
            raise ValueError("SymmArena supports 1..8 peers (one NVSwitch domain)")
        self.rank = 0 if self.single else int(rank)
        self.devices = list(devices) if self.single else [torch.device(device if device is not None else torch.cuda.current_device()).index or 0]
        self.offsets: dict[str, tuple[int, int, torch.dtype]] = {}
        off = _ALIGN  # control page first
        for name, (numel, dt) in planes.items():
            if dt not in _DT:
                raise ValueError(f"unsupported plane dtype {dt}")
            self.offsets[name] = (off, int(numel), dt)
            off = _round_up(off + int(numel) * _DT[dt][1], _ALIGN)
        self.nbytes = off
        self.epoch = 0
        self.mc_base = 0            # base of the NVLS multicast mapping of the arena (0 = not available)
        self._symm: Any = None
        self._group: Any = None
        self._opened: list[int] = []
        if self.single:
            for a in self.devices:
                for b in self.devices:
                    if a != b and not self.ext.enable_peer_access(a, b):
                        raise RuntimeError(f"GPU {a} cannot access GPU {b} (no P2P)")
            self.base = [self.ext.ipc_alloc(self.nbytes, dv) for dv in self.devices]
            self._owned = list(self.base)
        else:
            dv = self.devices[0]
            if self.world_size > 1 and self._try_nvls(dv, group):
                self._owned = []
                return
            mine = self.ext.ipc_alloc(self.nbytes, dv)
            self._owned = [mine]
            if self.world_size == 1:
                self.base = [mine]
            else:
                handles: list[Any] = [None] * self.world_size
                dist.all_gather_object(handles, bytes(self.ext.ipc_get_handle(mine)), group=group)
                self.base = []
                for r, hnd in enumerate(handles):
                    if r == self.rank:
                        self.base.append(mine)
                    else:
                        ptr = self.ext.ipc_open_handle(hnd, dv)
                        self._opened.append(ptr)
                        self.base.append(ptr)
                dist.barrier(group=group)

    def _try_nvls(self, dv: int, group: Any) -> bool:
        """Allocate the arena as torch symmetric memory with a multicast mapping; all ranks agree on the outcome."""
        ok, t, hdl = 0, None, None
        if os.environ.get("PB_NVLS", "1") != "0":
            try:
                import torch.distributed._symmetric_memory as symm_mem

                pg = group if group is not None else dist.group.WORLD
                t = symm_mem.empty(self.nbytes, dtype=torch.uint8, device=torch.device("cuda", dv))
                t.zero_()
                torch.cuda.synchronize(dv)
                hdl = symm_mem.rendezvous(t, group=pg.group_name)
                ok = int(bool(getattr(hdl, "multicast_ptr", 0)) and len(hdl.buffer_ptrs) == self.world_size)
            except Exception as e:  # noqa: BLE001 - any failure means "use the IPC path"
                print(f"[symm] NVLS arena unavailable ({type(e).__name__}: {str(e)[:120]}); using CUDA IPC + P2P", flush=True)
                ok = 0
        flag = torch.tensor([ok], device=torch.device("cuda", dv))
        dist.all_reduce(flag, op=dist.ReduceOp.MIN, group=group)
        if int(flag.item()) != 1:
            return False
        self._symm = (t, hdl)
        self._group = group
        self.base = [int(p) for p in hdl.buffer_ptrs]
        self.mc_base = int(hdl.multicast_ptr)
        dist.barrier(group=group)
        return True

    def mc_ptr(self, name: str) -> int:
        """Multicast address of a plane, or 0 = use the P2P loops: no NVLS mapping, or fewer than ``PB_NVLS_MIN_WORLD``
        (default 4) GPUs: with 2 GPUs the P2P loops move one peer read per element, from 4 GPUs on their traffic grows N-fold
        while the in-switch reduction's stays constant. Where the two cross over on a given system is not measured here; the
        variable moves the threshold."""
        if not self.mc_base or self.world_size < int(os.environ.get("PB_NVLS_MIN_WORLD", "4")):
            return 0
        return self.mc_base + self.offsets[name][0]

    # ------------------------------------------------------------------ views / pointers
    def _dev(self, rank: int | None) -> int:
        return self.devices[rank if (self.single and rank is not None) else 0]

    def plane(self, name: str, rank: int | None = None) -> torch.Tensor:
        """Torch view of a plane. In distributed mode only the local rank's plane is meant to be
        touched from torch; peers are reached from inside the kernels."""
        r = self.rank if rank is None else rank
        off, numel, dt = self.offsets[name]
        return self.ext.tensor_from_ptr(self.base[r] + off, numel, _DT[dt][0], self._dev(r))

    def ptrs(self, name: str) -> list[int]:
        off = self.offsets[name][0]
        return [b + off for b in self.base]

    def ctl_ptrs(self) -> list[int]:
        return list(self.base)

    def ctl_words(self, rank: int | None = None) -> torch.Tensor:
        r = self.rank if rank is None else rank
        return self.ext.tensor_from_ptr(self.base[r], self.ext.CTL_WORDS, "int32", self._dev(r))

    def ctl_sums(self, rank: int | None = None) -> torch.Tensor:
        """float64[8] by-products page: Σpg², Σa², Σx², Σm², Σv², -, -, scratch."""
        r = self.rank if rank is None else rank
        return self.ext.tensor_from_ptr(self.base[r] + 4 * self.ext.ctl_sums_word_offset(), 8, "float64", self._dev(r))

    def next_epoch(self) -> int:
        self.epoch += 1
        return self.epoch

    def shard(self, total: int, rank: int | None = None) -> tuple[int, int]:
        """Contiguous [lo,hi) slice of a flat index space owned by ``rank``; shards start on 256-element boundaries (the
        unit of the round kernel's per-tensor bookkeeping, and the alignment of every tensor in a FlatLayout)."""
        r = self.rank if rank is None else rank
        per = _round_up(-(-total // self.world_size), 256)
        lo = min(total, r * per)
        return lo, min(total, lo + per)

    def close(self) -> None:
        if self._symm is not None:
            # symmetric-memory arenas are not reference counted across ranks: nobody may free while a peer's kernel can still
            # touch this rank's pages (flag polling in the end barrier, multicast stores) -> collective teardown
            try:
                torch.cuda.synchronize(self.devices[0])
                if dist.is_initialized():
                    dist.barrier(group=self._group)
            except Exception:  # noqa: BLE001 - process group already gone at interpreter exit
                pass
        for p in self._opened:
            try:
                self.ext.ipc_close(p)
            except Exception:  # noqa: BLE001
                pass
        for p in self._owned:
            try:
                self.ext.ipc_free(p)
            except Exception:  # noqa: BLE001
                pass
        self._opened, self._owned = [], []
        self._symm = None
