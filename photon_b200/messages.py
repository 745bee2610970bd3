"""In-memory control-plane messages.

The reference moves these as Flower ``RecordSet``s over gRPC with every
non-scalar field stringified (ref: photon/server/server_util.py:205-302,
photon/client_app.py:182-211; SURVEY Appendix A).  The H100 engine keeps the
same *schema* (so logs, semantics and tests line up) but as plain dataclasses
passed through in-process / torch.distributed object channels — there is no
serialisation of tensors on either hot path: ``parameters`` is a handle (flat
tensor, shm metadata, or an NVLink arena slot), never bytes.
"""
from __future__ import annotations

import ast
from dataclasses import asdict, dataclass, field
from enum import IntEnum
from typing import Any


class Code(IntEnum):
    OK = 0
    GET_PROPERTIES_NOT_IMPLEMENTED = 1
    GET_PARAMETERS_NOT_IMPLEMENTED = 2
    FIT_NOT_IMPLEMENTED = 3
    EVALUATE_NOT_IMPLEMENTED = 4
    FAILED = 5


@dataclass
class Status:
    code: Code = Code.OK
    message: str = ""


@dataclass
class ClientState:
    """Per-client federation bookkeeping (ref: photon/utils.py:41-53)."""

    local_steps_cumulative: int = 0
    local_timestamp: dict[str, Any] = field(default_factory=dict)
    steps_done: int = 0

    def to_literal(self) -> dict[str, Any]:
        return asdict(self)

    @classmethod
    def from_literal(cls, d: dict[str, Any] | str) -> "ClientState":
        if isinstance(d, str):
            d = ast.literal_eval(d)
        return cls(**{k: d[k] for k in ("local_steps_cumulative", "local_timestamp", "steps_done") if k in d})


def encode_client_states(states: dict[int, ClientState]) -> str:
    """``str({cid: asdict(ClientState)})`` — the stringly wire form (ref: server_util.py:276-278)."""
    return str({int(c): s.to_literal() for c, s in states.items()})


def decode_client_states(s: str | dict[Any, Any]) -> dict[int, ClientState]:
    d = ast.literal_eval(s) if isinstance(s, str) else s
    return {int(c): ClientState.from_literal(v) for c, v in d.items()}


@dataclass
class ParamHandle:
    """Where a parameter payload lives. ``kind``: ``inline`` (flat torch tensor or list of
    ndarrays in ``data``), ``shm`` (POSIX segment name + metadata), ``nvl`` (arena slot id),
    ``file`` (npz path — the S3/object-store stand-in)."""

    kind: str = "inline"
    data: Any = None
    meta: dict[str, Any] = field(default_factory=dict)


@dataclass
class FitIns:
    parameters: ParamHandle | None
    config: dict[str, Any]


@dataclass
class FitRes:
    status: Status
    parameters: ParamHandle | None
    num_examples: int
    metrics: dict[str, Any] = field(default_factory=dict)
    cid: int | None = None


@dataclass
class EvaluateIns:
    parameters: ParamHandle | None
    config: dict[str, Any]


@dataclass
class EvaluateRes:
    status: Status
    loss: float
    num_examples: int
    metrics: dict[str, Any] = field(default_factory=dict)
    cid: int | None = None


@dataclass
class Message:
    """One control message: ``kind`` ∈ train | evaluate | query; ``content`` carries the
    Ins/Res object or a small dict (broadcast ack, free_resources …)."""

    kind: str
    content: Any
    node_id: int = 0
    group_id: str = "0"
    reply_to: int | None = None
    msg_id: int = 0
    error: str | None = None

    def has_content(self) -> bool:
        return self.content is not None and self.error is None
