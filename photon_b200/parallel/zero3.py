"""Full parameter sharding (ZeRO-3) inside a client / a centralised run: ``fsdp_config.sharding_strategy: FULL_SHARD``.

The reference hands this to PyTorch FSDP through Composer (ref: photon/conf/llm_config/mpt-7b.yaml:85-91): parameters, gradients
and optimizer state are sharded over the ranks, every block's parameters are all-gathered right before its forward / backward and
its gradient is reduce-scattered right after. Here, on one NVSwitch domain:

* the flat parameter index space is cut into UNITS (one per transformer block, one for embeddings + final norm and, for an untied
  LM head, one for ``lm_head.weight``, which sorts before the blocks); every unit
  is cut into ``world_size`` equal slices (256-aligned, zero padded) and rank r owns slice r of EVERY unit — so every gather and
  every reduction is balanced over the ranks whatever the unit (:class:`UnitPlan`, pure host logic);
* the persistent state of a rank is its shard only: fp32 masters and their bf16 copy (two planes of a :class:`SymmArena`, readable
  by peers), the fp32 gradient shard and the optimizer moments (16 B/param ÷ world_size instead of 18 B/param);
* **all-gather = the copy engines pull**: a unit's bf16 weights are assembled in one of two rotating local buffers with
  ``world_size`` peer-to-peer ``cudaMemcpyAsync`` calls on a side stream, one unit ahead of the compute stream — no SM is spent on
  it and NVSwitch gives every pull full bandwidth;
* **reduce-scatter = one fused NVLink kernel per unit** (``zero3_reduce_kernel``, csrc/comm.cu): the unit's gradient of this
  microbatch lands in a staging plane of the arena, every rank sums ITS slice over all ranks' staging planes (``multimem.ld_reduce``
  in the switch when NVLS is up) and accumulates the mean into its gradient shard;
* the optimizer is the same fused kernel as everywhere else, run on the shard (it is element-wise), writing fp32 masters and the
  bf16 copy peers will pull next step.

The 1-D parameters (LayerNorm gains, biases: < 0.1 % of the model) are needed in fp32 by the normalisation kernels: they are pulled
once per optimizer step from their owners' fp32 planes into a small resident buffer.

Under ``precision: amp_fp8`` (``NvlZero3Comm(..., fp8=True)``) the block GEMMs read E4M3 weights, so the block units are gathered
as E4M3 bytes (half the bf16 traffic) and no bf16 block buffers exist. Every parameter write already ends in
:meth:`NvlZero3Comm.params_changed`; there one ``zero3_fp8_requant_kernel`` per parameter version exchanges every block matrix's
amax over the ranks and lets each owner quantise its pieces of the matrix into an E4M3 shard plane, with the scale the unsharded
engine would compute from the whole tensor (bitwise the same bytes and scales). The embeddings / final norm and the 1-D
parameters are gathered as without fp8.
"""
from __future__ import annotations

import re
from dataclasses import dataclass
from typing import Any, Sequence

import numpy as np
import torch

from photon_b200.utils.flat import FlatLayout


def _round_up(x: int, m: int) -> int:
    return (x + m - 1) // m * m


# the weight matrices of every block, in the engine's weight-role order (the four fp8 GEMMs of a block)
BLOCK_MATRICES = ("attn.Wqkv.weight", "attn.out_proj.weight", "ffn.up_proj.weight", "ffn.down_proj.weight")


@dataclass(frozen=True)
class Unit:
    name: str           # "block.{i}", "rest" or "head"
    lo: int             # span [lo, hi) in the flat index space
    hi: int
    per: int            # slice length (multiple of 256); the padded span is world_size * per >= hi - lo
    off: int            # offset of this unit's slice inside every rank's shard


class UnitPlan:
    """Where every flat index lives: ``unit`` → (span, slice length, shard offset). Host-only arithmetic (unit-tested on CPU)."""

    def __init__(self, layout: FlatLayout, n_layers: int, world_size: int, align: int = 256) -> None:
        self.layout, self.world_size, self.n_layers = layout, int(world_size), int(n_layers)
        pat = re.compile(r"^transformer\.blocks\.(\d+)\.")
        first: dict[int, int] = {}
        last_block_end = 0
        for n, o, ne in zip(layout.names, layout.offsets, layout.numels):
            m = pat.match(n)
            if m:
                b = int(m.group(1))
                first[b] = min(first.get(b, o), o)
                last_block_end = max(last_block_end, _round_up(o + ne, layout.align))
        if sorted(first) != list(range(n_layers)):
            raise ValueError(f"layout holds blocks {sorted(first)}, expected 0..{n_layers - 1}")
        starts = sorted(first.values())
        # tensors that sort before the first block (an untied lm_head.weight) form the "head" unit
        head_end = starts[0]
        if any(o < head_end and o + ne > head_end for o, ne in zip(layout.offsets, layout.numels)):
            raise ValueError("a tensor straddles the start of the transformer blocks in the flat layout")
        ends = {s: (starts[k + 1] if k + 1 < len(starts) else last_block_end) for k, s in enumerate(starts)}
        units, off = [], 0
        for b in range(n_layers):               # numeric order = execution order
            lo, hi = first[b], ends[first[b]]
            per = _round_up(-(-(hi - lo) // self.world_size), align)
            units.append(Unit(f"block.{b}", lo, hi, per, off))
            off += per
        lo, hi = last_block_end, layout.total
        per = _round_up(-(-(hi - lo) // self.world_size), align)
        units.append(Unit("rest", lo, hi, per, off))
        off += per
        # appended after "rest": block i stays unit i, and a layout without tensors before the blocks plans as it always did
        self.head: int | None = None
        if head_end > 0:
            per = _round_up(-(-head_end // self.world_size), align)
            self.head = len(units)
            units.append(Unit("head", 0, head_end, per, off))
            off += per
        self.units: list[Unit] = units
        self.shard_len = off
        self.max_block_span = max(u.per for u in units[:n_layers]) * self.world_size
        self.rest_span = units[n_layers].per * self.world_size
        self.head_span = units[self.head].per * self.world_size if self.head is not None else 0
        # tensor -> unit
        self.unit_of: list[int] = []
        for n, o in zip(layout.names, layout.offsets):
            m = pat.match(n)
            self.unit_of.append(int(m.group(1)) if m else self.head if o < head_end else n_layers)
        # 1-D parameters, packed: (tensor index, offset in the packed fp32 buffer)
        self.small_index: dict[str, int] = {}
        self.small_offsets: dict[str, int] = {}
        soff = 0
        for i, (n, shp, ne) in enumerate(zip(layout.names, layout.shapes, layout.numels)):
            if len(shp) <= 1:
                self.small_index[n], self.small_offsets[n] = i, soff
                soff = _round_up(soff + ne, 64)
        self.small_len = max(soff, 64)

    @property
    def rest(self) -> int:
        return self.n_layers

    def resident_unit(self, u: int) -> bool:
        """Units held whole in a resident buffer (embeddings + final norm, the untied head) rather than a rotating one."""
        return u == self.rest or u == self.head

    def rel(self, name: str) -> tuple[int, int, int]:
        """(unit index, offset inside the unit's padded span, numel) of a tensor."""
        i = self.layout.index(name)
        u = self.unit_of[i]
        return u, self.layout.offsets[i] - self.units[u].lo, self.layout.numels[i]

    def slice_range(self, u: int, r: int) -> tuple[int, int]:
        """Flat range covered by slice ``r`` of unit ``u`` (clipped to the unit; may be empty)."""
        un = self.units[u]
        lo = min(un.hi, un.lo + r * un.per)
        return lo, min(un.hi, lo + un.per)

    # -- full <-> shard (host or device tensors) -------------------------------------------------------
    def full_to_shard(self, full: torch.Tensor, rank: int, out: torch.Tensor) -> torch.Tensor:
        """``out`` (shard_len) = rank's slices of ``full`` (layout.total), zero padded."""
        out.zero_()
        for u, un in enumerate(self.units):
            lo, hi = self.slice_range(u, rank)
            if hi > lo:
                out[un.off: un.off + hi - lo].copy_(full[lo:hi])
        return out

    def shard_to_full(self, shard: torch.Tensor, rank: int, full: torch.Tensor) -> torch.Tensor:
        """Scatter rank's slices into ``full`` (other positions untouched)."""
        for u, un in enumerate(self.units):
            lo, hi = self.slice_range(u, rank)
            if hi > lo:
                full[lo:hi].copy_(shard[un.off: un.off + hi - lo])
        return full

    def small_copies(self) -> list[tuple[int, int, int, int]]:
        """(owner rank, offset in the owner's shard, offset in the packed small buffer, n) for every piece of every 1-D tensor."""
        out = []
        for n, i in self.small_index.items():
            u = self.unit_of[i]
            un = self.units[u]
            pos, left, dst = self.layout.offsets[i] - un.lo, self.layout.numels[i], self.small_offsets[n]
            while left > 0:
                r = pos // un.per
                k = min(left, (r + 1) * un.per - pos)
                out.append((r, un.off + pos - r * un.per, dst, k))
                pos, left, dst = pos + k, left - k, dst + k
        return out

    # -- block weight matrices (amp_fp8: their E4M3 copies are quantised piecewise by the owners) --------
    @property
    def weight_names(self) -> list[str]:
        """Block weight matrices in slot order: block by block, :data:`BLOCK_MATRICES` within a block."""
        return [f"transformer.blocks.{i}.{m}" for i in range(self.n_layers) for m in BLOCK_MATRICES]

    def weight_pieces(self, rank: int) -> list[tuple[int, int, int]]:
        """(offset in ``rank``'s shard, numel, weight slot) of every non-empty piece of every block weight matrix inside that
        rank's slices. A matrix meets one slice in at most one contiguous piece; offsets and lengths are multiples of 8 (the
        kernel moves 8 elements per vector access)."""
        out = []
        for j, name in enumerate(self.weight_names):
            u, rel, n = self.rel(name)
            un = self.units[u]
            if rel % 8 or n % 8:
                raise ValueError(f"{name}: offset / size must be multiples of 8 for the E4M3 weight shards")
            lo, hi = max(rel, rank * un.per), min(rel + n, (rank + 1) * un.per)
            if hi > lo:
                out.append((un.off + lo - rank * un.per, hi - lo, j))
        return out

    def bytes_per_rank(self, n_moments: int = 2, fp8: bool = False) -> dict[str, int]:
        """Persistent + transient device bytes of one rank (the memory table in DESIGN.md). ``fp8``: the block units travel as
        E4M3 (no bf16 block buffers) and the E4M3 shard plane, the amax planes and this rank's partial amax are added. An untied
        head unit adds its resident bf16 buffer and fp32 staging plane (bf16 under fp8 too)."""
        S = self.shard_len
        out = {"masters_fp32": 4 * S, "bf16_copy": 2 * S, "grad_shard_fp32": 4 * S, "moments_fp32": 4 * n_moments * S,
               "unit_weight_buffers_bf16": 2 * 2 * self.max_block_span + 2 * self.rest_span + 2 * self.head_span,
               "grad_staging_fp32": 4 * 2 * self.max_block_span + 4 * self.rest_span + 4 * self.head_span,
               "small_fp32": 4 * self.small_len}
        if fp8:
            n_w = len(self.weight_names)
            out.update(unit_weight_buffers_bf16=2 * self.rest_span + 2 * self.head_span, e4m3_shard=S,
                       unit_weight_buffers_e4m3=2 * self.max_block_span,
                       amax_fp32=4 * (self.world_size + 1) * n_w)
        return out


class ShardedFlat:
    """What the optimizer, the trainer and the checkpoints see instead of :class:`FlatParams` under ZeRO-3: ``params`` / ``grads``
    are this rank's SHARD (the optimizer is element-wise), ``full_params`` / ``load_full_params`` assemble / distribute the whole
    vector on demand (checkpoints, parameter loads — never on the step path)."""

    is_sharded = True

    def __init__(self, comm: "NvlZero3Comm") -> None:
        self.comm, self.layout = comm, comm.plan.layout
        self.params, self.grads = comm.p32, comm.gshard

    @property
    def names(self) -> tuple[str, ...]:
        return self.layout.names

    def zero_grad(self) -> None:
        self.grads.zero_()

    def full_params(self) -> torch.Tensor:
        return self.comm.gather_full_params()

    def load_full_params(self, full: torch.Tensor) -> None:
        self.comm.load_full_params(full)

    def to_ndarrays(self) -> list[np.ndarray]:
        return self.layout.to_ndarrays(self.full_params())

    def load_ndarrays(self, arrays: Sequence[np.ndarray]) -> None:
        full = torch.zeros(self.layout.total, dtype=torch.float32)
        self.layout.from_ndarrays(full, arrays)
        self.load_full_params(full)


class NvlZero3Comm:
    """Arena, buffers, streams and the gather / reduce schedule of one rank. The engine asks for views (``weight`` / ``weight8`` /
    ``small`` / ``grad``) once at bind time and calls ``acquire`` / ``prefetch`` / ``reduce`` around every block."""

    zero3 = True

    def __init__(self, layout: FlatLayout, n_layers: int, *, rank: int, world_size: int, device: torch.device | int | None = None,
                 group: Any = None, fp8: bool = False) -> None:
        """``fp8``: the engine runs ``precision: amp_fp8`` — block units are gathered as E4M3 from a shard plane that
        :meth:`params_changed` requantises (after :meth:`attach_fp8`), instead of as bf16."""
        from photon_b200 import ops
        from photon_b200.parallel.symm import SymmArena

        self.ext = ops.ext()
        self.plan = UnitPlan(layout, n_layers, world_size)
        self.rank, self.world_size, self.group = int(rank), int(world_size), group
        self.fp8 = bool(fp8)
        pl = self.plan
        planes = {"p32": (pl.shard_len, torch.float32), "w16": (pl.shard_len, torch.bfloat16),
                  "gs0": (pl.max_block_span, torch.float32), "gs1": (pl.max_block_span, torch.float32),
                  "gsr": (pl.rest_span, torch.float32)}
        if pl.head is not None:
            planes["gsh"] = (pl.head_span, torch.float32)
        if self.fp8:
            self._pieces = pl.weight_pieces(self.rank)
            self.n_weights = len(pl.weight_names)
            planes.update(w8=(pl.shard_len, torch.uint8), amax=(self.world_size * self.n_weights, torch.float32))
        self.arena = SymmArena(planes, rank=rank, world_size=world_size, device=device, group=group)
        self.dev = torch.device("cuda", self.arena.devices[0])
        ar = self.arena
        self.p32, self.w16 = ar.plane("p32"), ar.plane("w16")
        self.p32.zero_(), self.w16.zero_()
        self.gstage = [ar.plane("gs0"), ar.plane("gs1")]
        self.gstage_rest = ar.plane("gsr")
        self.gstage_head = ar.plane("gsh") if pl.head is not None else None
        self.gshard = torch.zeros(pl.shard_len, dtype=torch.float32, device=self.dev)
        self.wbuf: list[torch.Tensor] | None = None         # bf16 block units (without fp8)
        self.wbuf8: list[torch.Tensor] | None = None        # E4M3 block units (fp8)
        self._fp8_meta: torch.Tensor | None = None
        if self.fp8:
            self.w8, self.amax = ar.plane("w8"), ar.plane("amax")
            self.w8.zero_(), self.amax.zero_()
            self.amax_local = torch.zeros(self.n_weights, dtype=torch.float32, device=self.dev)
            self.pieces = torch.tensor(self._pieces, dtype=torch.int64).reshape(-1, 3).to(self.dev)
            self.wbuf8 = [torch.zeros(pl.max_block_span, dtype=torch.uint8, device=self.dev) for _ in range(2)]
        else:
            self.wbuf = [torch.zeros(pl.max_block_span, dtype=torch.bfloat16, device=self.dev) for _ in range(2)]
        self.wrest = torch.zeros(pl.rest_span, dtype=torch.bfloat16, device=self.dev)
        # the untied LM head: resident and bf16, also under fp8 (the head GEMMs stay bf16)
        self.whead = torch.zeros(pl.head_span, dtype=torch.bfloat16, device=self.dev) if pl.head is not None else None
        self.small32 = torch.zeros(pl.small_len, dtype=torch.float32, device=self.dev)
        self._small_copies = pl.small_copies()
        self.side = torch.cuda.Stream(self.dev)
        self.resident: list[int | None] = [None, None]      # unit held (or being pulled into) each rotating buffer
        self._ready: list[Any] = [None, None]               # event: the pull into buffer k has finished
        self._rest_valid = False
        self.version = 0                                     # bumped whenever the parameters change (cached whole-model copies key on it)
        self.norm = torch.zeros(1, dtype=torch.float32, device=self.dev)

    # ------------------------------------------------------------------ views for the engine
    def weight(self, name: str) -> torch.Tensor | None:
        """bf16 view of a gathered weight; None for a block matrix under fp8 (its GEMMs read :meth:`weight8`)."""
        u, rel, n = self.plan.rel(name)
        if not self.plan.resident_unit(u) and self.wbuf is None:
            return None
        buf = self.wrest if u == self.plan.rest else self.whead if u == self.plan.head else self.wbuf[u % 2]
        return buf[rel: rel + n].view(self.plan.layout.shapes[self.plan.layout.index(name)])

    def weight8(self, name: str) -> torch.Tensor:
        """E4M3 view of a gathered block weight matrix (fp8 only)."""
        u, rel, n = self.plan.rel(name)
        if self.wbuf8 is None or self.plan.resident_unit(u):
            raise ValueError(f"{name}: E4M3 weights exist for the block matrices of an fp8 communicator only")
        return self.wbuf8[u % 2][rel: rel + n].view(self.plan.layout.shapes[self.plan.layout.index(name)])

    def attach_fp8(self, meta: torch.Tensor, roles: Sequence[int]) -> None:
        """The engine's fp8 scaling state ``meta`` [3, n_roles] and the role column of every weight slot
        (:attr:`UnitPlan.weight_names` order): from now on :meth:`params_changed` requantises the weights and writes their
        scale / 1/scale / amax there."""
        if not self.fp8:
            raise ValueError("attach_fp8 needs NvlZero3Comm(..., fp8=True)")
        if len(roles) != self.n_weights:
            raise ValueError(f"expected {self.n_weights} weight roles, got {len(roles)}")
        self._fp8_meta = meta
        self._roles = torch.tensor(list(roles), dtype=torch.int32, device=self.dev)

    def requantize(self) -> None:
        """One ``zero3_fp8_requant_kernel``: every rank's E4M3 shard and the weight scales from the current bf16 shards (a
        collective: every rank calls it, in the same order as the other collectives of this communicator)."""
        ar = self.arena
        self.ext.zero3_fp8_requant(ar.ctl_ptrs(), ar.rank, ar.devices[0], ar.next_epoch(), self.w16, self.w8, self.pieces,
                                   self.amax_local, ar.ptrs("amax"), self._fp8_meta, self._roles)

    def small(self, name: str) -> torch.Tensor:
        i, o = self.plan.small_index[name], self.plan.small_offsets[name]
        return self.small32[o: o + self.plan.layout.numels[i]].view(self.plan.layout.shapes[i])

    def _stage(self, u: int) -> torch.Tensor:
        return self.gstage_rest if u == self.plan.rest else self.gstage_head if u == self.plan.head else self.gstage[u % 2]

    def grad(self, name: str) -> torch.Tensor:
        u, rel, n = self.plan.rel(name)
        buf = self._stage(u)
        return buf[rel: rel + n].view(self.plan.layout.shapes[self.plan.layout.index(name)])

    # ------------------------------------------------------------------ all-gather (copy-engine pulls)
    def _pull(self, dst: torch.Tensor, plane: str, off: int, per: int, esize: int) -> None:
        src = self.arena.ptrs(plane)
        for r in range(self.world_size):
            self.ext.memcpy_async(dst.data_ptr() + r * per * esize, src[r] + off * esize, per * esize, self.dev.index)

    def _issue(self, u: int) -> None:
        """Pull unit ``u`` into buffer ``u % 2`` on the side stream, after everything enqueued so far on the compute stream (the
        previous tenant of the buffer has been consumed by then)."""
        k, un = u % 2, self.plan.units[u]
        self.side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.cuda.stream(self.side):
            if self.fp8:
                self._pull(self.wbuf8[k], "w8", un.off, un.per, 1)
            else:
                self._pull(self.wbuf[k], "w16", un.off, un.per, 2)
            ev = torch.cuda.Event()
            ev.record(self.side)
        self.resident[k], self._ready[k] = u, ev

    def prefetch(self, u: int) -> None:
        if 0 <= u < self.plan.n_layers and self.resident[u % 2] != u:
            self._issue(u)

    def acquire(self, u: int) -> None:
        """The compute stream may read unit ``u`` after this returns (stream-ordered; the host does not block)."""
        k = u % 2
        if self.resident[k] != u:
            self._issue(u)
        if self._ready[k] is not None:
            torch.cuda.current_stream(self.dev).wait_event(self._ready[k])

    def ensure_resident(self) -> None:
        """Embeddings + final norm (bf16), the untied head (bf16) and every 1-D parameter (fp32): pulled once per parameter
        version."""
        if self._rest_valid:
            return
        un = self.plan.units[self.plan.rest]
        self._pull(self.wrest, "w16", un.off, un.per, 2)
        if self.plan.head is not None:
            un = self.plan.units[self.plan.head]
            self._pull(self.whead, "w16", un.off, un.per, 2)
        src = self.arena.ptrs("p32")
        for r, soff, doff, n in self._small_copies:
            self.ext.memcpy_async(self.small32.data_ptr() + 4 * doff, src[r] + 4 * soff, 4 * n, self.dev.index)
        self._rest_valid = True

    # ------------------------------------------------------------------ reduce-scatter (fused NVLink kernel)
    def zero_stage(self, u: int) -> None:
        self._stage(u).zero_()

    def reduce(self, u: int) -> None:
        un, ar = self.plan.units[u], self.arena
        plane = "gsr" if u == self.plan.rest else "gsh" if u == self.plan.head else ("gs0", "gs1")[u % 2]
        self.ext.zero3_reduce(ar.ctl_ptrs(), ar.rank, ar.devices[0], ar.next_epoch(), ar.ptrs(plane), ar.mc_ptr(plane),
                              self.gshard[un.off: un.off + un.per], un.per)

    def barrier(self) -> None:
        ar = self.arena
        self.ext.zero3_reduce(ar.ctl_ptrs(), ar.rank, ar.devices[0], ar.next_epoch(), [], 0, None, 0)

    # ------------------------------------------------------------------ parameter versions
    def before_param_write(self) -> None:
        """Nobody may still be pulling the old parameters from this rank when they are overwritten."""
        torch.cuda.current_stream(self.dev).wait_stream(self.side)
        self.barrier()

    def params_changed(self) -> None:
        """Every rank's new shard is in place before anybody pulls from it; local copies of the old version are dropped. Under
        fp8 (once attached) the requantisation kernel takes the place of the barrier: it ends with the same one."""
        if self._fp8_meta is not None:
            self.requantize()
        else:
            self.barrier()
        self.resident, self._ready = [None, None], [None, None]
        self._rest_valid = False
        self.version += 1

    def all_reduce_mean_(self, g: torch.Tensor) -> torch.Tensor:
        return g        # every unit was reduced (and averaged) right after its backward

    def grad_norm(self, g: torch.Tensor) -> torch.Tensor:
        """‖gradient‖₂ over ALL shards (device scalar)."""
        from photon_b200 import ops

        sq = ops.flat_l2_norm(g).square().reshape(1)
        if self.world_size > 1:
            import torch.distributed as dist

            dist.all_reduce(sq, group=self.group)
        return sq.sqrt()[0]

    # ------------------------------------------------------------------ whole-vector access (never on the step path)
    def gather_full_params(self) -> torch.Tensor:
        """fp32 ``[layout.total]`` on this rank's device, pulled slice by slice from the owners."""
        pl = self.plan
        full = torch.zeros(pl.layout.total, dtype=torch.float32, device=self.dev)
        tmp = torch.empty(max(pl.max_block_span, pl.rest_span, pl.head_span), dtype=torch.float32, device=self.dev)
        torch.cuda.current_stream(self.dev).wait_stream(self.side)
        for un in pl.units:
            self._pull(tmp, "p32", un.off, un.per, 4)
            full[un.lo: un.hi].copy_(tmp[: un.hi - un.lo])
        return full

    def load_full_params(self, full: torch.Tensor) -> None:
        """Every rank passes the SAME full vector (host or device); each keeps its slices."""
        from photon_b200 import ops

        self.before_param_write()
        shard = torch.zeros(self.plan.shard_len, dtype=torch.float32, device="cpu" if full.device.type == "cpu" else self.dev)
        self.plan.full_to_shard(full, self.rank, shard)
        self.p32.copy_(shard)
        ops.cast_bf16(self.p32, self.w16)
        self.params_changed()

    def close(self) -> None:
        self.arena.close()
