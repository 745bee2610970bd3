"""Typed schema for the resolved config tree.

Same key surface as the reference's ``BaseConfig`` (ref:
photon/conf/base_schema.py:11-392) plus two H100-native additions:
``photon.comm_stack.nvl`` (fused NVLink kernels for the round hot paths) and
the optional ``kernels`` section (which hand-written sm_90a ops are on).
Validation is strict on the federation/photon nodes and permissive on
``llm_config`` / ``dataset`` (free-form in the reference too, ref:
base_schema.py:336-342).
"""
from __future__ import annotations

from enum import Enum
from typing import Any

from pydantic import BaseModel, ConfigDict, Field, field_validator, model_validator


class _Strict(BaseModel):
    model_config = ConfigDict(extra="forbid")


class CommStack(_Strict):
    """Bulk-tensor transport for the two round hot paths (exactly one on)."""

    s3: bool = False
    shm: bool = True
    ray: bool = False
    nvl: bool = False  # H100-native: in-kernel NVLink P2P / multicast path

    @model_validator(mode="after")
    def _one_hot(self) -> "CommStack":
        on = [k for k in ("s3", "shm", "ray", "nvl") if getattr(self, k)]
        if len(on) != 1:
            raise ValueError(f"exactly one comm stack must be enabled, got {on or 'none'}")
        return self

    @property
    def active(self) -> str:
        return next(k for k in ("nvl", "shm", "ray", "s3") if getattr(self, k))


class Centralized(_Strict):
    store_init_model: bool = False
    store_final_model: bool = False
    stream_id: int | str | None = None
    eval_only: bool = False
    split_eval: bool = False
    reset_timestamp: bool = False


class Fleet(_Strict):
    """Cross-host nodes of ``photon.topology=nodes`` (photon_b200/server/grpc_fleet.py): the server listens on ``address`` and waits
    for ``n_remote_nodes`` machines running ``python -m photon_b200.node --server host:port``."""

    address: str | None = None            # host:port the fleet link binds (null = every interface, an ephemeral port — printed at start)
    n_remote_nodes: int = 0
    liveness_timeout_s: float = 30.0      # a node that has not polled for this long is gone (its client goes to another node)
    connect_timeout_s: float = 600.0      # how long the server waits for the remote nodes to register
    # hierarchical aggregation: a node keeps the weighted sum of the clients it trained in a round and ships ONE model when the
    # server collects (instead of one per client, as the reference does) — the same global model, 1/clients-per-node of the traffic
    node_pre_aggregation: bool = False


class Photon(_Strict):
    n_nodes: int = 1                      # in-process nodes of topology=nodes (0 = the server machine trains nothing itself)
    fleet: Fleet = Field(default_factory=Fleet)
    task_timeout_s: float | None = None   # node manager: presume the workers hung after this long without a result (null = wait forever)
    topology: str = "spmd"   # spmd: one process per GPU + fused round transports; nodes: server → ClientApp → NodeManager → Workers
    refresh_period: int = 50
    checkpoint: bool = False
    restore_run_uuid: str | None = None
    restore_cent_run_uuid: str | None = None
    restore_cent_run_batches: int | None = None
    copy_client_checkpoints: bool = True
    resume_round: int | None = -1
    saving_path: str | None = None
    comm_stack: CommStack = Field(default_factory=CommStack)
    # SPMD host control plane (photon_b200/server/control.py): liveness, shared work queue, time-bounded metadata exchange
    client_state_cache_device_gb: float = 16.0   # per-client optimizer moments kept between participations: on the GPU up to this,
    client_state_cache_host_gb: float = 64.0     # then in pinned host memory up to this, then the least recently used client is dropped
    async_checkpoint: bool = True         # server checkpoints: snapshot at the round boundary, write on a background thread
    control_plane: str = "store"          # store | none
    scheduling: str = "dynamic"           # dynamic = shared work queue (a free GPU takes the next client) | static = client i -> node i mod n
    liveness_timeout_s: float = 20.0      # a rank whose heartbeat is older than this is dead
    progress_timeout_s: float = 900.0     # a rank whose main thread made no progress for this long stops its heartbeat (hung = dead)
    kernel_peer_timeout_s: float = 120.0  # bound on every cross-GPU spin inside the NVLink kernels (aborted round instead of a hang)

    @field_validator("refresh_period")
    @classmethod
    def _positive(cls, v: int) -> int:
        if v < 1:
            raise ValueError("must be >= 1")
        return v

    @field_validator("n_nodes")
    @classmethod
    def _non_negative(cls, v: int) -> int:
        if v < 0:
            raise ValueError("must be >= 0")
        return v

    @field_validator("topology")
    @classmethod
    def _topology(cls, v: str) -> str:
        if v not in ("spmd", "nodes"):
            raise ValueError("photon.topology must be 'spmd' or 'nodes'")
        return v


class StrategyName(str, Enum):
    """Server optimizers (ref: base_schema.py:100-137, strategy/dispatcher.py:44-165).
    ``nestorov`` keeps the reference's spelling; ``nesterov`` is accepted too."""

    NESTOROV = "nestorov"
    FEDMOM = "fedmom"
    FEDAVG = "fedavg"
    FEDYOGI = "fedyogi"
    FEDADAM = "fedadam"

    @classmethod
    def parse(cls, v: Any) -> "StrategyName":
        if isinstance(v, cls):
            return v
        s = str(v).strip().lower()
        if s == "nesterov":
            s = "nestorov"
        return cls(s)


class FL(_Strict):
    n_total_clients: int = 8
    n_clients_per_round: int = 8
    n_rounds: int = 200
    reset_checkpoint: bool = False
    reset_optimizer: bool = True
    reset_dataset_state: bool = False
    reset_timestamp: bool = False
    resize_vocab: int | None = None
    use_unigram_metrics: bool = False
    allow_unigram_metrics_failures: bool = False
    n_local_epochs: int = 1
    n_local_steps: int = 0
    random_layers: list[str] = Field(default_factory=list)
    random_init_freq: int = 0
    truly_random_init: bool = True
    personalized_layers: list[str] = Field(default_factory=list)
    frozen_layers: list[str] | None = None
    unfrozen_layers: list[str] | None = None
    ignore_failed_rounds: bool = False
    accept_failures_cnt: int = 0
    eval_period: int | None = 1
    split_eval: bool = False
    strategy_name: StrategyName = StrategyName.NESTOROV
    strategy_kwargs: dict[str, Any] = Field(default_factory=dict)
    set_trainer_params_filter_keys: bool = True
    set_trainer_key_to_filter: str = "transformer"
    aggregate_momenta: bool = False
    use_noise_scale_metric: bool = False
    noise_scale_beta: float = 0.99
    # H100-native additions (absent keys default to reference behaviour)
    reference_sign_compat: bool = False  # FedAdam/FedYogi ascent quirk, SURVEY §2.4
    fault_injection: dict[str, Any] | None = None  # {"round": r, "cid": k, "kind": "drop"}

    @field_validator("strategy_name", mode="before")
    @classmethod
    def _strategy(cls, v: Any) -> StrategyName:
        return StrategyName.parse(v)

    @model_validator(mode="after")
    def _check(self) -> "FL":
        if not 1 <= self.n_clients_per_round <= self.n_total_clients:
            raise ValueError("need 1 <= n_clients_per_round <= n_total_clients")
        if self.frozen_layers and self.unfrozen_layers:
            # ref: photon/clients/trainer_utils.py:1173-1177
            raise ValueError("frozen_layers and unfrozen_layers are mutually exclusive")
        return self


class ClientConfig(BaseModel):
    """Time-outs of the S3 client (ref: base_schema.py:236-247); extra botocore keys are accepted and ignored."""

    model_config = {"extra": "allow"}
    connect_timeout: float = 3600
    read_timeout: float = 3600


class BackendKwargs(BaseModel):
    """(ref: base_schema.py:250-262) + what the own S3 client reads: ``endpoint_url`` (else ``S3_ENDPOINT_URL``), ``region_name``
    (else ``AWS_DEFAULT_REGION``), ``prefix`` inside the bucket."""

    model_config = {"extra": "allow"}
    client_config: ClientConfig = Field(default_factory=ClientConfig)
    endpoint_url: str | None = None
    region_name: str | None = None
    prefix: str | None = None


class S3CommConfig(_Strict):
    bucket_name: str = "checkpoints"
    num_attempts: int = 3
    backend_kwargs: BackendKwargs = Field(default_factory=BackendKwargs)


class StrategyKWArgs(dict):       # noqa: FURB189 - free-form mappings, named like the reference's schema nodes (ref: base_schema.py:138,336,340)
    """``fl.strategy_kwargs``: whatever the chosen server optimizer takes."""


class Dataset(dict):              # noqa: FURB189
    """``dataset``: the train / val stream tables (validated by the loaders)."""


class LLMConfig(dict):            # noqa: FURB189
    """``llm_config``: the Composer / llm-foundry style trainer node (validated where it is consumed)."""


class WandbSetup(BaseModel):
    model_config = ConfigDict(extra="allow")
    project: str = "photon"
    group: str = "llm"
    tags: list[str] = Field(default_factory=list)
    entity: str | None = None
    mode: str = "online"
    name: str | None = None
    resume: str = "allow"
    id: str | None = None
    allow_val_change: bool = True


class Wandb(_Strict):
    setup: WandbSetup = Field(default_factory=WandbSetup)


class Kernels(_Strict):
    """Which hand-written sm_90a kernels the engine uses (H100-native knob).
    ``auto`` = on when a CUDA device is present, plain PyTorch on CPU."""

    gemm: str = "auto"        # wgmma/TMA GEMM family
    attention: str = "auto"   # wgmma flash attention
    norm: str = "auto"        # fused residual+LayerNorm
    loss: str = "auto"        # fused cross-entropy
    optimizer: str = "auto"   # fused flat-buffer ADOPT / DecoupledAdamW
    cuda_graph: bool = True
    # sharding inside a client / a centralised run when fsdp_config asks for it: zero1 = optimizer state only (one fused NVLink
    # step), zero3 = parameters + gradients + state (parallel/zero3.py), auto = zero3 only when the model would crowd the GPU
    param_sharding: str = "auto"

    @field_validator("param_sharding")
    @classmethod
    def _sharding(cls, v: str) -> str:
        if v not in ("auto", "zero1", "zero3"):
            raise ValueError("must be one of auto|zero1|zero3")
        return v

    @field_validator("gemm", "attention", "norm", "loss", "optimizer")
    @classmethod
    def _mode(cls, v: str) -> str:
        if v not in ("auto", "b200", "torch"):
            raise ValueError("must be one of auto|b200|torch")
        return v


class BaseConfig(BaseModel):
    """Root (ref: base_schema.py:344-392)."""

    model_config = ConfigDict(extra="forbid")
    run_uuid: str
    seed: int = 1337
    pretrained_model_path: str | None = None
    wte_parameters_path: str | None = None
    cleanup_checkpoints: bool = False
    cleanup_checkpoints_per_round: bool = False
    use_wandb: bool = False
    centralized: Centralized = Field(default_factory=Centralized)
    photon: Photon = Field(default_factory=Photon)
    fl: FL = Field(default_factory=FL)
    s3_comm_config: S3CommConfig = Field(default_factory=S3CommConfig)
    wandb: Wandb = Field(default_factory=Wandb)
    kernels: Kernels = Field(default_factory=Kernels)
    llm_config: dict[str, Any]
    dataset: dict[str, Any]
    eval_gauntlet_config: dict[str, Any] | None = None
    icl_tasks_config: dict[str, Any] | None = None

    @field_validator("run_uuid", mode="before")
    @classmethod
    def _uuid(cls, v: Any) -> str:
        return str(v)

    @model_validator(mode="after")
    def _llm(self) -> "BaseConfig":
        llm = self.llm_config
        for key in ("model", "optimizer", "max_seq_len", "global_train_batch_size", "precision"):
            if key not in llm:
                raise ValueError(f"llm_config.{key} is required")
        prec = llm["precision"]
        if prec not in ("amp_bf16", "amp_fp16", "fp32", "amp_fp8"):
            raise ValueError(f"llm_config.precision={prec!r} unsupported")
        if llm.get("tp_config") not in (None, {}):
            # TP is plumbing-only in the reference and never enabled (SURVEY §2.6)
            raise ValueError("llm_config.tp_config must be null")
        impl = llm["model"].get("attn_config", {}).get("attn_impl", "flash")
        if impl not in ("flash", "torch", "b200"):
            raise ValueError(f"attn_impl={impl!r} unsupported (flash|torch|b200)")
        return self


def register_config(name: str = "base_schema") -> None:
    """The reference registers its schema with Hydra's ConfigStore so YAML files can name it in ``defaults``
    (ref: base_schema.py:395-398). The own composer validates every composed config against :class:`BaseConfig` anyway
    (``validate_config``), so there is nothing to register; kept so ``register_config("base_schema")`` call sites keep working."""
    del name


def validate_config(cfg: Any) -> BaseConfig:
    """Validate a composed tree; raises ``pydantic.ValidationError`` on mismatch."""
    from photon_b200.config.composer import to_container

    return BaseConfig.model_validate(to_container(cfg))
