"""POSIX shared-memory codecs for the host hand-off path.

Role of ref photon/shm/utils.py (:138-651): model parameters travel between the
node manager, its workers and the server as ONE flat segment described by
``ModelParametersMetadata`` (per-tensor byte bounds, shapes, dtypes); scalars
(n_samples int64, eval loss float64) and pickled dicts (configs, metrics) get
their own tiny segments.  On the H100 path this is the *fallback / baseline*
transport (``photon.comm_stack.shm``) — the product path is the NVLink arena —
but it is also what the CPU plumbing tests and the multi-process node manager use.

Differences from the reference, on purpose: segments are unregistered from
Python's resource tracker through the public ``track=False`` flag where
available (instead of monkey-patching, ref :403-429) and ``close_all_shms``
removes every suffixed segment of a uuid (the reference leaks them, SURVEY App. D #5).
"""
from __future__ import annotations

import pickle
import sys
import threading
from dataclasses import asdict, dataclass, field
from multiprocessing import shared_memory
from typing import Any, Sequence

import numpy as np

from photon_b200.shm import constants as C


# The resource tracker keeps a SET of names per process tree: two threads attaching the same segment concurrently
# would interleave register/register/unregister/unregister and the second unregister raises inside the tracker.
# Attach + untrack (and open + unlink) therefore run under one process-wide lock.
_TRACKER_LOCK = threading.RLock()


def _open(name: str, create: bool = False, size: int = 0, untrack: bool = True) -> shared_memory.SharedMemory:
    kw: dict[str, Any] = {}
    if sys.version_info >= (3, 13):
        kw["track"] = False
    with _TRACKER_LOCK:
        shm = shared_memory.SharedMemory(name=name, create=create, size=size if create else 0, **kw)
        if sys.version_info < (3, 13) and untrack:
            remove_shm_from_resource_tracker(shm)
    return shm


def remove_shm_from_resource_tracker(shm: shared_memory.SharedMemory) -> None:
    """Detach the segment from the creating process' resource tracker so it survives that
    process (the consumer unlinks it)."""
    try:
        from multiprocessing import resource_tracker

        resource_tracker.unregister(shm._name, "shared_memory")  # type: ignore[attr-defined]  # noqa: SLF001
    except Exception:  # noqa: BLE001
        pass


def shm_exists(name: str) -> bool:
    try:
        s = _open(name)
    except FileNotFoundError:
        return False
    s.close()
    return True


def unlink_quietly(name: str) -> None:
    with _TRACKER_LOCK:
        try:
            s = _open(name, untrack=False)  # stays registered so that unlink()'s unregister is balanced
        except FileNotFoundError:
            return
        s.close()
        try:
            s.unlink()
        except FileNotFoundError:
            pass


@dataclass
class ModelParametersMetadata:
    """Layout of a flat parameter segment (ref: shm/utils.py:138-247)."""

    total_num_bytes: int = 0
    array_bounds: list[tuple[int, int]] = field(default_factory=list)
    shapes: list[tuple[int, ...]] = field(default_factory=list)
    dtypes: list[str] = field(default_factory=list)

    @classmethod
    def from_ndarrays(cls, arrays: Sequence[np.ndarray], align: int = 64) -> "ModelParametersMetadata":
        bounds, shapes, dtypes, off = [], [], [], 0
        for a in arrays:
            a = np.asarray(a)
            lo = (off + align - 1) // align * align
            hi = lo + a.nbytes
            bounds.append((lo, hi)), shapes.append(tuple(a.shape)), dtypes.append(str(a.dtype))
            off = hi
        return cls(total_num_bytes=max(off, 1), array_bounds=bounds, shapes=shapes, dtypes=dtypes)

    def to_literal(self) -> str:
        return str(asdict(self))

    @classmethod
    def from_literal(cls, s: str | dict[str, Any]) -> "ModelParametersMetadata":
        import ast

        d = ast.literal_eval(s) if isinstance(s, str) else s
        return cls(total_num_bytes=int(d["total_num_bytes"]), array_bounds=[tuple(b) for b in d["array_bounds"]],
                   shapes=[tuple(x) for x in d["shapes"]], dtypes=list(d["dtypes"]))

    def same_layout(self, other: "ModelParametersMetadata") -> bool:
        return self.shapes == other.shapes and self.dtypes == other.dtypes


def set_parameters_shm(name: str, arrays: Sequence[np.ndarray], meta: ModelParametersMetadata | None = None,
                       create: bool = True) -> tuple[shared_memory.SharedMemory, ModelParametersMetadata]:
    """Write ``arrays`` into segment ``name`` (created if missing). Caller keeps the handle alive."""
    meta = meta or ModelParametersMetadata.from_ndarrays(arrays)
    try:
        shm = _open(name)
        if shm.size < meta.total_num_bytes:
            shm.close()
            unlink_quietly(name)
            raise FileNotFoundError
    except FileNotFoundError:
        if not create:
            raise
        shm = _open(name, create=True, size=meta.total_num_bytes)
    for a, (lo, hi), shp, dt in zip(arrays, meta.array_bounds, meta.shapes, meta.dtypes):
        dst = np.ndarray(shp, dtype=np.dtype(dt), buffer=shm.buf[lo:hi])
        np.copyto(dst, np.asarray(a, dtype=np.dtype(dt)).reshape(shp))
    return shm, meta


def get_parameters_shm(name: str, meta: ModelParametersMetadata, copy: bool = False
                       ) -> tuple[shared_memory.SharedMemory, list[np.ndarray]]:
    """Zero-copy per-tensor views over segment ``name`` (ref: shm/utils.py:569-623).
    Keep the returned handle referenced for as long as the views are used."""
    shm = _open(name)
    views = [np.ndarray(shp, dtype=np.dtype(dt), buffer=shm.buf[lo:hi])
             for (lo, hi), shp, dt in zip(meta.array_bounds, meta.shapes, meta.dtypes)]
    if copy:
        views = [v.copy() for v in views]
    return shm, views


# ----------------------------------------------------------------------------- scalars
def _scalar(name: str, dtype: str, value: Any | None) -> Any:
    nbytes = np.dtype(dtype).itemsize
    if value is not None:
        try:
            shm = _open(name)
        except FileNotFoundError:
            shm = _open(name, create=True, size=nbytes)
        np.ndarray((1,), dtype=dtype, buffer=shm.buf[:nbytes])[0] = value
        shm.close()
        return value
    shm = _open(name)
    out = np.ndarray((1,), dtype=dtype, buffer=shm.buf[:nbytes])[0].item()
    shm.close()
    return out


def set_n_samples_shm(uuid: str, n: int) -> None:
    _scalar(uuid + C.W_N_SAMPLES_SHM, "int64", int(n))


def get_n_samples_shm(uuid: str) -> int:
    return int(_scalar(uuid + C.W_N_SAMPLES_SHM, "int64", None))


def set_eval_loss_shm(uuid: str, loss: float) -> None:
    _scalar(uuid + C.W_EVAL_LOSS_SHM, "float64", float(loss))


def get_eval_loss_shm(uuid: str) -> float:
    return float(_scalar(uuid + C.W_EVAL_LOSS_SHM, "float64", None))


# --------------------------------------------------------------------- pickled dict segments
def set_dict_shm(name: str, obj: Any) -> None:
    """8-byte length header + pickle payload; the segment is re-created when it must grow."""
    blob = pickle.dumps(obj, protocol=pickle.HIGHEST_PROTOCOL)
    need = 8 + len(blob)
    try:
        shm = _open(name)
        if shm.size < need:
            shm.close()
            unlink_quietly(name)
            raise FileNotFoundError
    except FileNotFoundError:
        shm = _open(name, create=True, size=max(need, 4096))
    shm.buf[:8] = len(blob).to_bytes(8, "little")
    shm.buf[8:need] = blob
    shm.close()


def get_dict_shm(name: str) -> Any:
    shm = _open(name)
    n = int.from_bytes(bytes(shm.buf[:8]), "little")
    obj = pickle.loads(bytes(shm.buf[8:8 + n]))  # noqa: S301 - same-host IPC between our own processes
    shm.close()
    return obj


def close_all_shms(uuid: str) -> None:
    """Unlink every segment this uuid may own (bare + all suffixes)."""
    for suffix in ("", C.NM_CONFIG_SHM, C.NM_PARAMS_SHM, C.W_PARAMS_SHM, C.W_N_SAMPLES_SHM, C.W_EVAL_LOSS_SHM, C.W_METRICS_SHM):
        unlink_quietly(uuid + suffix)


# ----------------------------------------------------------------------------- reference-shaped forms (ref: photon/shm/utils.py)
# The reference's helpers hand back (view, SharedMemory) pairs the caller keeps mapped; these do the same on top of ``_open``.
def is_shm_existing(name: str) -> bool:
    """(ref: shm/utils.py:525-545)"""
    return shm_exists(name)


def get_ndarrays_size_and_bounds(ndarrays: Sequence[np.ndarray]) -> tuple[int, list[tuple[int, int]]]:
    """Total bytes of a parameter payload and the [start, end) byte range of every array inside one flat segment
    (ref: shm/utils.py:104-140)."""
    bounds, off = [], 0
    for a in ndarrays:
        n = int(np.asarray(a).nbytes)
        bounds.append((off, off + n))
        off += n
    return off, bounds


def get_num_samples_shm(name: str, *, create: bool = False) -> tuple[np.ndarray, shared_memory.SharedMemory]:
    """A mapped one-element int64 array — the sample count a worker reports (ref: shm/utils.py:271-309)."""
    shm = _open(name, create=create, size=8) if create else _open(name)
    view = np.ndarray((1,), dtype=np.int64, buffer=shm.buf[:8])
    if create:
        view[0] = 0
    return view, shm


def set_num_samples_shm(old_num_samples_sh: np.ndarray, new_num_samples: int) -> None:
    """(ref: shm/utils.py:312-330)"""
    old_num_samples_sh[0] = int(new_num_samples)


def _pickled_segment(obj: Any, name: str, create: bool) -> tuple[Any, shared_memory.SharedMemory]:
    if create:
        set_dict_shm(name, obj)
    shm = _open(name)
    n = int.from_bytes(bytes(shm.buf[:8]), "little")
    return pickle.loads(bytes(shm.buf[8:8 + n])), shm  # noqa: S301 - same-host IPC between our own processes


def _store_pickled(obj: Any, shm: shared_memory.SharedMemory) -> None:
    blob = pickle.dumps(obj, protocol=pickle.HIGHEST_PROTOCOL)
    if 8 + len(blob) > shm.size:
        raise ValueError(f"object needs {8 + len(blob)} bytes, the segment holds {shm.size}: re-create it with get_*_shm(create=True)")
    shm.buf[:8] = len(blob).to_bytes(8, "little")
    shm.buf[8:8 + len(blob)] = blob


def get_config_shm(config: Any, name: str, *, create: bool = False) -> tuple[Any, shared_memory.SharedMemory]:
    """The run config through a named segment: ``create=True`` publishes ``config``, otherwise it is read back
    (ref: shm/utils.py:477-522)."""
    return _pickled_segment(config, name, create)


def set_config_shm(config: Any, shm: shared_memory.SharedMemory) -> None:
    """(ref: shm/utils.py:548-568)"""
    _store_pickled(config, shm)


def get_dict_configsrecord_shm(name: str, config: Any = None, *, create: bool = False) -> tuple[Any, shared_memory.SharedMemory]:
    """A dict of per-client instruction records (fit / evaluate configs) through a named segment (ref: shm/utils.py:432-474)."""
    return _pickled_segment(config, name, create)


def set_dict_configsrecord_shm(config: Any, shm: shared_memory.SharedMemory) -> None:
    """(ref: shm/utils.py:250-268)"""
    _store_pickled(config, shm)
