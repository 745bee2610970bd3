"""Multi-stream, rank-partitioned, resumable token dataset + loader.

Covers what the reference gets from mosaicml-streaming's ``StreamingDataset``
and llm-foundry's text dataloader (ref: photon/clients/llm_config_functions.py:
239-606 stream selection + dataset defaults; SURVEY App. C "Text dataloader" /
"Streaming"): streams mixed by ``proportion`` / ``repeat`` / ``choose``,
deterministic shuffle (seed 9176 by default), partitioning over ranks, a
``state_dict`` that resumes mid-epoch (the ``*dataset_state*`` checkpoint key)
and a collator producing ``{"input_ids", "labels"}`` LongTensors of fully
packed sequences.  A stream whose ``local`` is ``synthetic://...`` (or whose
directory does not exist while ``allow_synthetic``) is backed by
:class:`SyntheticC4`, because this environment has no real C4.
"""
from __future__ import annotations

import os
import sys
import queue
import zlib
import threading
from dataclasses import dataclass
from pathlib import Path
from typing import Any, Iterator, Sequence

import numpy as np
import torch

from photon_b200.data.shards import INDEX_NAME, ShardReader, open_shard_dir
from photon_b200.data.synthetic import SyntheticC4

SYNTH_PREFIX = "synthetic://"


@dataclass
class Stream:
    """One entry of ``client_streams`` (ref: conf/dataset/streams/*.yaml)."""

    local: str | None = None
    remote: str | None = None
    split: str | None = None
    proportion: float | None = None
    repeat: float | None = None
    choose: int | None = None
    download_retry: int | None = None
    download_timeout: float | None = None
    validate_hash: str | None = None
    keep_zip: bool | None = None
    name: str = "stream"

    def directory(self) -> Path | None:
        if self.local is None or str(self.local).startswith(SYNTH_PREFIX):
            return None
        p = Path(self.local)
        return p / self.split if self.split else p


_WARNED_SYNTH: set[str] = set()


def _open_stream(st: Stream, seq_len: int, idx: int, synth_samples: int, seed: int, allow_synthetic: bool,
                 synth_vocab: int | None = None) -> Any:
    d = st.directory()
    if d is not None and (d / INDEX_NAME).exists():
        return open_shard_dir(d, validate_hash=bool(st.validate_hash))   # our shards, or an MDS directory written for the reference
    strict = os.environ.get("PHOTON_STRICT_DATA", "").lower() in ("1", "true", "yes")   # the launch scripts export it for real runs
    if d is not None and (strict or not allow_synthetic):
        raise FileNotFoundError(f"stream '{st.name}': {d} has no {INDEX_NAME} (and remote fetch is unavailable offline); "
                                "use local: synthetic://<name> for synthetic tokens")
    if d is not None and str(d) not in _WARNED_SYNTH:
        # a typo or an unmounted dataset must not train on synthetic tokens unnoticed
        _WARNED_SYNTH.add(str(d))
        print(f"[streaming] WARNING: stream '{st.name}': {d} has no {INDEX_NAME} -> SYNTHETIC C4-shaped tokens are used instead. "
              "Set dataset.<split>.allow_synthetic=false or PHOTON_STRICT_DATA=1 to make this an error.", file=sys.stderr, flush=True)
    sid = idx
    if st.local and str(st.local).startswith(SYNTH_PREFIX):
        tail = str(st.local)[len(SYNTH_PREFIX):]
        sid = int(tail) if tail.isdigit() else (zlib.crc32(tail.encode()) % (1 << 30))  # stable across processes
    elif st.local:
        digits = "".join(ch for ch in Path(str(st.local)).name if ch.isdigit())
        sid = int(digits) if digits else idx
    kw = {"vocab_size": int(synth_vocab)} if synth_vocab else {}   # never emit ids the (possibly resized) model cannot embed
    return SyntheticC4(seq_len=seq_len, seed=seed, stream_id=sid, num_samples=_synthetic_split_size(st.split, synth_samples), **kw)


# a synthetic stand-in is as long as the split it replaces would be (documents of the truncated C4 splits; ref:
# photon/dataset/constants/mc4.py:39-44,67-72) so that "evaluate on val_xxsmall" stays a seconds-long job
_SYNTH_SPLIT_SAMPLES = {"val_xxsmall": 100, "val_xsmall": 3_000, "val_small": 10_000, "val": 1 << 14, "validation": 1 << 14}


def _synthetic_split_size(split: str | None, default: int) -> int:
    return min(default, _SYNTH_SPLIT_SAMPLES.get(str(split), default)) if split else default


class StreamingTokenDataset:
    """Epoch-wise sampler over N streams.

    Per epoch each stream contributes ``choose`` samples (explicit, or
    ``repeat × len``, or by ``proportion`` of ``epoch_size``); the concatenated
    id list is optionally shuffled with ``shuffle_seed + epoch`` and rank ``r``
    of ``w`` takes ids ``r, r+w, …`` (equal count on every rank → DDP-safe).
    """

    def __init__(self, streams: Sequence[Stream | dict[str, Any]], seq_len: int = 2048, *, shuffle: bool = False,
                 shuffle_seed: int = 9176, epoch_size: int | None = None, rank: int = 0, world_size: int = 1,
                 synthetic_samples: int = 1 << 16, synthetic_seed: int = 17, allow_synthetic: bool = True,
                 synthetic_vocab: int | None = None, **_unused: Any) -> None:
        self.streams = [s if isinstance(s, Stream) else Stream(**{k: v for k, v in s.items() if k in Stream.__annotations__})
                        for s in streams]
        if not self.streams:
            raise ValueError("need at least one stream")
        self.seq_len, self.shuffle, self.shuffle_seed = int(seq_len), bool(shuffle), int(shuffle_seed)
        self.rank, self.world_size, self.epoch_size = int(rank), int(world_size), epoch_size
        self._sources = [_open_stream(s, self.seq_len, i, synthetic_samples, synthetic_seed, allow_synthetic, synthetic_vocab)
                         for i, s in enumerate(self.streams)]
        for src in self._sources:
            if getattr(src, "seq_len", self.seq_len) != self.seq_len:
                raise ValueError(f"stream seq_len {src.seq_len} != requested {self.seq_len}")
        self._counts = self._per_stream_counts()
        self.epoch = 0
        self.sample_in_epoch = 0  # per-rank position

    def _per_stream_counts(self) -> list[int]:
        lens = [len(s) for s in self._sources]
        if any(s.proportion is not None for s in self.streams):
            props = np.array([float(s.proportion or 0.0) for s in self.streams])
            props = props / props.sum()
            total = self.epoch_size or sum(lens)
            return [int(round(total * p)) for p in props]
        counts = []
        for s, n in zip(self.streams, lens):
            if s.choose is not None:
                counts.append(int(s.choose))
            elif s.repeat is not None:
                counts.append(int(round(n * float(s.repeat))))
            else:
                counts.append(n)
        if self.epoch_size:
            scale = self.epoch_size / max(1, sum(counts))
            counts = [max(1, int(c * scale)) for c in counts]
        return counts

    def _epoch_ids(self, epoch: int) -> np.ndarray:
        parts = []
        for si, (c, src) in enumerate(zip(self._counts, self._sources)):
            n = len(src)
            ids = np.arange(c, dtype=np.int64) % n
            if c < n and self.shuffle:  # sub-sample without replacement, epoch-dependent
                ids = np.random.default_rng([self.shuffle_seed, epoch, si]).choice(n, size=c, replace=False)
            parts.append(np.stack([np.full(c, si, dtype=np.int64), ids], axis=1))
        allids = np.concatenate(parts, axis=0)
        if self.shuffle:
            allids = allids[np.random.default_rng([self.shuffle_seed, epoch]).permutation(len(allids))]
        usable = len(allids) // self.world_size * self.world_size
        return allids[:usable][self.rank::self.world_size]

    def samples_per_epoch(self) -> int:
        return sum(self._counts) // self.world_size

    def __iter__(self) -> Iterator[np.ndarray]:
        while True:
            ids = self._epoch_ids(self.epoch)
            while self.sample_in_epoch < len(ids):
                si, ix = ids[self.sample_in_epoch]
                self.sample_in_epoch += 1
                yield self._sources[int(si)][int(ix)]
            self.epoch += 1
            self.sample_in_epoch = 0
            return  # one epoch per iterator, like a sized torch DataLoader

    def state_dict(self) -> dict[str, int]:
        return {"epoch": self.epoch, "sample_in_epoch": self.sample_in_epoch,
                "world_size": self.world_size, "shuffle_seed": self.shuffle_seed}

    def load_state_dict(self, sd: dict[str, int]) -> None:
        self.epoch = int(sd.get("epoch", 0))
        pos = int(sd.get("sample_in_epoch", 0))
        old_w = int(sd.get("world_size", self.world_size))
        self.sample_in_epoch = pos * old_w // self.world_size  # elastic resume across world sizes


def sequence_ids(ids: torch.Tensor, eos_token_id: int | None = None, bos_token_id: int | None = None) -> torch.Tensor | None:
    """llm-foundry's ``sequence_id`` of a packed batch ``[B, S]``: the document index of every token, counted from 0 in each
    row. EOS mode: ``cumsum(ids == eos)`` shifted right by one, so the EOS token belongs to the document it ends. BOS mode:
    ``cumsum(ids == bos)``, so the BOS token opens its document. None when neither id is given."""
    if eos_token_id is not None and bos_token_id is not None:
        raise ValueError("Cannot use both eos_token_id and bos_token_id to detect document boundaries")
    if bos_token_id is not None:
        return torch.cumsum(ids == int(bos_token_id), dim=1).to(ids.dtype)
    if eos_token_id is None:
        return None
    cs = torch.cumsum(ids == int(eos_token_id), dim=1).to(ids.dtype)
    return torch.cat([cs.new_zeros(cs.shape[0], 1), cs[:, :-1]], dim=1)


class TokenLoader:
    """Batches a :class:`StreamingTokenDataset` into pinned ``[B,S]`` int64 tensors.
    ``num_workers>0`` turns on a background prefetch thread (host side only; the H2D
    copy belongs to the trainer's copy stream)."""

    def __init__(self, dataset: StreamingTokenDataset, batch_size: int, drop_last: bool = True,
                 num_workers: int = 0, prefetch: int = 4, pin_memory: bool | None = None,
                 eos_token_id: int | None = None, bos_token_id: int | None = None) -> None:
        """``eos_token_id`` / ``bos_token_id`` (at most one; llm-foundry's ``dataset`` keys): add a per-token ``sequence_id``
        to every batch that numbers the documents of each packed row (see :func:`sequence_ids`)."""
        if eos_token_id is not None and bos_token_id is not None:
            raise ValueError("Cannot use both eos_token_id and bos_token_id to detect document boundaries")
        self.dataset, self.batch_size, self.drop_last = dataset, int(batch_size), bool(drop_last)
        self.eos_token_id, self.bos_token_id = eos_token_id, bos_token_id
        self.num_workers, self.prefetch = int(num_workers), int(prefetch)
        self.pin = torch.cuda.is_available() if pin_memory is None else pin_memory
        # position of the CONSUMER (the trainer), not of the producer: the prefetch thread runs ahead of what has been
        # trained on, so a checkpoint must not store the dataset's own cursor (mosaicml-streaming derives its
        # ``state_dict`` from the number of samples the trainer has seen for the same reason)
        self._live: tuple[int, int] | None = None   # (epoch, sample_in_epoch) at the start of the running iterator
        self._handed_out = 0                         # batches the consumer has received from it

    def __len__(self) -> int:
        n = self.dataset.samples_per_epoch()
        return n // self.batch_size if self.drop_last else -(-n // self.batch_size)

    def _collate(self, rows: list[np.ndarray]) -> dict[str, torch.Tensor]:
        ids = torch.from_numpy(np.stack(rows).astype(np.int64))
        sid = sequence_ids(ids, self.eos_token_id, self.bos_token_id)
        if self.pin:
            ids = ids.pin_memory()
            sid = sid.pin_memory() if sid is not None else None
        batch = {"input_ids": ids, "labels": ids}  # labels == inputs; the shift happens in the loss
        if sid is not None:
            batch["sequence_id"] = sid
        return batch

    def _gen(self) -> Iterator[dict[str, torch.Tensor]]:
        rows: list[np.ndarray] = []
        for r in self.dataset:
            rows.append(r)
            if len(rows) == self.batch_size:
                yield self._collate(rows)
                rows = []
        if rows and not self.drop_last:
            yield self._collate(rows)

    def __iter__(self) -> Iterator[dict[str, torch.Tensor]]:
        self._live, self._handed_out = (self.dataset.epoch, self.dataset.sample_in_epoch), 0
        it = self._iter_batches()
        try:
            for batch in it:
                self._handed_out += 1
                yield batch
        finally:
            it.close()   # stops and joins the prefetch thread before the cursor is rewound
            # exhausted (the dataset already points at the next epoch) or abandoned: its own cursor is authoritative again
            if self._live is not None and self.dataset.epoch == self._live[0]:
                self.dataset.sample_in_epoch = self._live[1] + self._handed_out * self.batch_size   # drop what was only prefetched
            self._live = None

    def _iter_batches(self) -> Iterator[dict[str, torch.Tensor]]:
        if self.num_workers <= 0:
            yield from self._gen()
            return
        q: "queue.Queue[Any]" = queue.Queue(maxsize=self.prefetch)
        stop = threading.Event()

        def work() -> None:
            try:
                for b in self._gen():
                    while not stop.is_set():
                        try:
                            q.put(b, timeout=0.1)
                            break
                        except queue.Full:
                            continue
                    if stop.is_set():
                        return
                q.put(None)
            except BaseException as e:  # noqa: BLE001 - forwarded to the consumer
                q.put(e)

        th = threading.Thread(target=work, daemon=True, name="pb200-prefetch")
        th.start()
        try:
            while True:
                item = q.get()
                if item is None:
                    return
                if isinstance(item, BaseException):
                    raise item
                yield item
        finally:
            stop.set()
            th.join(timeout=5.0)

    def state_dict(self) -> dict[str, int]:
        sd = self.dataset.state_dict()
        if self._live is not None:
            sd["epoch"], sd["sample_in_epoch"] = self._live[0], self._live[1] + self._handed_out * self.batch_size
        return sd

    def load_state_dict(self, sd: dict[str, int]) -> None:
        self.dataset.load_state_dict(sd)
        self._live = None


def build_text_loader(loader_cfg: dict[str, Any], batch_size: int, rank: int = 0, world_size: int = 1,
                      seed: int = 17, vocab_size: int | None = None) -> TokenLoader:
    """``loader_cfg`` = ``llm_config.train_loader`` / ``eval_loader`` after the client-side
    stream surgery has replaced ``dataset.streams`` with a flat ``{name: Stream-dict}`` map
    (ref: photon/clients/llm_config_functions.py:239-529)."""
    ds_cfg = dict(loader_cfg.get("dataset", {}) or {})
    streams_cfg = ds_cfg.pop("streams", None) or {}
    split = ds_cfg.pop("split", None)
    root_local = ds_cfg.pop("root_local", None) or ds_cfg.pop("local", None)
    ds_cfg.pop("root_remote", None)
    # llm-foundry's text collator keys: either one makes every batch carry a per-token sequence_id
    eos_token_id, bos_token_id = ds_cfg.pop("eos_token_id", None), ds_cfg.pop("bos_token_id", None)
    if eos_token_id is not None and bos_token_id is not None:
        raise ValueError("dataset: set at most one of eos_token_id and bos_token_id")
    streams: list[Stream] = []
    if isinstance(streams_cfg, dict):
        for name, sc in streams_cfg.items():
            sc = dict(sc or {})
            local = sc.get("local")
            if local is not None and root_local and not str(local).startswith((SYNTH_PREFIX, "/")):
                local = os.path.join(root_local, local)
            elif local is None:
                local = root_local
            streams.append(Stream(**{**{k: v for k, v in sc.items() if k in Stream.__annotations__},
                                     "local": local, "split": sc.get("split", split), "name": str(name)}))
    if not streams:
        streams = [Stream(local=root_local, split=split, name="default")]
    nw = loader_cfg.get("num_workers", 0)
    ds = StreamingTokenDataset(streams, seq_len=int(ds_cfg.pop("max_seq_len", 2048)),
                               shuffle=bool(ds_cfg.pop("shuffle", False)),
                               shuffle_seed=int(ds_cfg.pop("shuffle_seed", 9176) or 9176),
                               epoch_size=ds_cfg.pop("epoch_size", None), rank=rank, world_size=world_size,
                               synthetic_seed=seed, synthetic_vocab=vocab_size,
                               **{k: v for k, v in ds_cfg.items() if k in ("synthetic_samples", "allow_synthetic")})
    return TokenLoader(ds, batch_size=batch_size, drop_last=bool(loader_cfg.get("drop_last", True)),
                       num_workers=0 if nw in (None, "auto") else min(int(nw), 1),
                       eos_token_id=eos_token_id, bos_token_id=bos_token_id)
