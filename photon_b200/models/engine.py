"""B200Engine (name kept for compatibility) — the MPT training step on hand-written sm_90a kernels.

No autograd, no per-op dispatcher: forward and backward are an explicit
schedule of our own kernels over preallocated bf16 activations, flat fp32
master parameters/gradients and a flat bf16 compute shadow
(SURVEY §2.5 (a) K1–K15 → one engine):

* every linear layer = ``csrc/gemm_tcgen05.cu`` (TMA → wgmma → register
  accumulators → fused epilogue): bias, bias+residual, bias+GELU (pre-activation and
  activation written by the same epilogue), dgrad with the stored weight
  consumed MN-major (no transposes), dGELU fused into the dgrad epilogue, wgrad
  with both operands MN-major accumulating in fp32 by red.global.add straight
  into the flat gradient bucket that the DDP all-reduce / optimizer consume;
* LM head + cross-entropy chunked over tokens so the ``[T, 50368]`` logits are
  never materialised (``[chunk, V]`` scratch that stays L2/HBM friendly);
  the chunk's dlogits feed the dgrad/wgrad GEMMs immediately;
* LayerNorm / RMSNorm fwd/bwd (+ residual-gradient add), embedding gather/scatter,
  bias-gradient column sums, loss statistics: ``csrc/fused_ops.cu``;
* attention: ``csrc/attention_tcgen05.cu`` (``attention: b200``) or, when
  ``kernels.attention: torch``, cuDNN/FA2 SDPA as an explicit library fallback.

The module tree of :class:`MPTForCausalLM` is kept only as the *owner of names
and initial values*: its parameters are views into the flat fp32 buffer, so the
federated payload / checkpoint order (sorted names) is shared with the torch
backend and the two are directly comparable in tests.
"""
from __future__ import annotations

from typing import Any

import torch
import torch.nn.functional as F

from photon_b200 import ops
from photon_b200.models.mpt import (MPTConfig, MPTForCausalLM, check_sequence_id, ffn_desc, nondefault_ffn, shift_labels,
                                    window_keep)
from photon_b200.train.backend import apply_freeze
from photon_b200.utils.flat import FlatLayout, FlatParams

# One block's backward as stages in execution order, each with the parameters whose gradients it produces (a stage's input
# gradient feeds the next one; the residual path joins at ln2 / ln1). "ln2" / "ln1" and the q/k norms of "attn" (the attention
# backward with them) are LayerNorms or RMSNorms (cfg.norm_type). Names absent from a layout are never trainable: a norm's bias
# under RMSNorm or no_bias, and the gate projection ("up" covers it in a gated FFN) in an mptmlp one.
BLOCK_STAGES = (("down", ("ffn.down_proj.weight", "ffn.down_proj.bias")),
                ("up", ("ffn.up_proj.weight", "ffn.up_proj.bias", "ffn.gate_proj.weight", "ffn.gate_proj.bias")),
                ("ln2", ("norm_2.weight", "norm_2.bias")),
                ("out", ("attn.out_proj.weight", "attn.out_proj.bias")),
                ("attn", ("attn.q_ln.weight", "attn.q_ln.bias", "attn.k_ln.weight", "attn.k_ln.bias")),
                ("qkv", ("attn.Wqkv.weight", "attn.Wqkv.bias")),
                ("ln1", ("norm_1.weight", "norm_1.bias")))


class BackwardPlan:
    """Which parts of the backward run, given the trainable parameter names (a pure function of the config and that set).

    The backward is one chain of stages: LM head, final LayerNorm, the blocks from the last down to the first
    (:data:`BLOCK_STAGES` each), embeddings. The head stage owns ``transformer.wte.weight`` when the head is tied (``tied``) and
    ``lm_head.weight`` otherwise; ``wte`` then belongs to the embedding stage only. A stage runs when it, or any stage after it, has a trainable parameter; its input
    gradient (the dgrad GEMM, the LayerNorm dx) is computed only when a later stage has one. So the backward stops right after the
    last stage that produces a trainable gradient, and weight / bias / LayerNorm-parameter gradients run for trainable names
    only. With every parameter trainable this is the full schedule."""

    def __init__(self, n_layers: int, trainable: Any, tied: bool = True) -> None:
        self.n_layers = int(n_layers)
        self.trainable = frozenset(trainable)
        self.head_weight = "transformer.wte.weight" if tied else "lm_head.weight"
        t = lambda names, pre="transformer.": any(pre + n in self.trainable for n in names)  # noqa: E731
        chain = [("head", t((self.head_weight,), "")), ("norm_f", t(("norm_f.weight", "norm_f.bias")))]
        for i in range(self.n_layers - 1, -1, -1):
            chain += [((i, s), t(names, f"transformer.blocks.{i}.")) for s, names in BLOCK_STAGES]
        chain.append(("embed", t(("wte.weight", "wpe.weight"))))
        self._pos = {k: j for j, (k, _) in enumerate(chain)}
        self.last = max((j for j, (_, has) in enumerate(chain) if has), default=-1)   # the last stage that runs

    def runs(self, stage: Any) -> bool:
        """``stage``: "head", "norm_f", "embed" or ``(block, name)`` with a name of :data:`BLOCK_STAGES`."""
        return self._pos[stage] <= self.last

    def dx(self, stage: Any) -> bool:
        """Whether the stage computes the gradient of its input (some stage after it needs it)."""
        return self._pos[stage] < self.last

    def grad(self, name: str) -> bool:
        return name in self.trainable

    @property
    def head_wgrad(self) -> bool:
        return self.grad(self.head_weight)

    @property
    def lowest_block(self) -> int:
        """The lowest block whose backward runs (``n_layers`` when none does)."""
        return next((i for i in range(self.n_layers) if self.runs((i, BLOCK_STAGES[0][0]))), self.n_layers)

    def block_stages(self, i: int) -> list[str]:
        return [s for s, _ in BLOCK_STAGES if self.runs((i, s))]


class _LayerW:
    """Per-block handles: bf16 weights (shadow plane), fp32 small params and fp32 grads."""

    __slots__ = ("wqkv", "bqkv", "wo", "bo", "wup", "bup", "wdown", "bdown", "g1", "b1", "g2", "b2",
                 "d_wqkv", "d_bqkv", "d_wo", "d_bo", "d_wup", "d_bup", "d_wdown", "d_bdown", "d_g1", "d_b1", "d_g2", "d_b2",
                 "qk_g", "qk_b", "d_qk_g", "d_qk_b", "wgate", "bgate", "d_wgate", "d_bgate")


class B200Engine:
    kind = "b200"

    def __init__(self, cfg: MPTConfig, device: torch.device | str = "cuda", precision: str = "amp_bf16",
                 kernels: dict[str, Any] | None = None, seed: int | None = 17, frozen_layers: list[str] | None = None,
                 unfrozen_layers: list[str] | None = None, unigram_log_probs: torch.Tensor | None = None,
                 lm_head_chunk: int = 16896, grads_storage: torch.Tensor | None = None,
                 activation_checkpointing: bool = False, params_storage: torch.Tensor | None = None,
                 shadow_storage: torch.Tensor | None = None, zero3: Any = None) -> None:
        """``zero3``: a :class:`photon_b200.parallel.zero3.NvlZero3Comm` — full parameter sharding: this rank keeps 1/world of the
        masters / gradients / bf16 weights, block weights are pulled into two rotating buffers one block ahead of the compute
        stream and every block's gradient is reduce-scattered right after its backward (ref: fsdp_config FULL_SHARD). Under
        ``amp_fp8`` it must be built with ``fp8=True``: the block weights then travel as E4M3 (see :meth:`_init_fp8`)."""
        self.cfg = cfg
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("B200Engine needs a CUDA (sm_90a) device")
        if precision not in ("amp_bf16", "amp_fp8"):
            raise NotImplementedError(f"B200Engine computes in bf16 (got precision={precision}); use kernels.*=torch for fp32/fp16")
        if (frozen_layers or unfrozen_layers) and zero3 is not None:
            raise NotImplementedError("freeze lists are not covered under full parameter sharding (kernels.*=torch runs them)")
        if nondefault_ffn(cfg) and (precision == "amp_fp8" or zero3 is not None):
            raise NotImplementedError(f"{ffn_desc(cfg)} is not covered under amp_fp8 or full parameter sharding "
                                      "(kernels.*=torch runs it)")
        if cfg.ffn_hidden % 8:
            # every GEMM operand / output row and the bias-gradient column sums of the FFN are [*, F] bf16 rows that must
            # be 16-byte multiples (the TMA row-stride and N % 8 launch checks)
            raise ValueError(f"the sm_90a engine needs an FFN width that is a multiple of 8, got {cfg.ffn_hidden}")
        ops.ext()  # fail loudly if the extension is missing
        self.precision = precision
        self.zero3 = zero3
        kernels = dict(kernels or {})
        # amp_fp8 (ref: scripts/centralised_training.sh:91, Composer amp_fp8 -> TransformerEngine): the four GEMMs of every block
        # and their dgrad / wgrad run on fp8 wgmma (E4M3 activations / weights, E5M2 gradients, per-tensor
        # scaling, accumulation in the tensor cores' reduced fp8 precision: tests/fp8_oracle.py); LayerNorm, attention, residuals,
        # LM head, loss and optimizer stay bf16 / fp32
        self.fp8 = precision == "amp_fp8"
        if zero3 is not None and bool(getattr(zero3, "fp8", False)) != self.fp8:
            raise ValueError(f"precision={precision} needs NvlZero3Comm(..., fp8={self.fp8}): block units are gathered as "
                             f"{'E4M3' if self.fp8 else 'bf16'}")
        self.attn_mode = "torch" if kernels.get("attention", "auto") == "torch" else "b200"
        # kernels.cuda_graph: the ~330 launches of one microbatch are captured once per (batch, seq, loss scaling) and
        # replayed (the schedule is static: preallocated workspace, TMA descriptors baked into the launches)
        # (not under full sharding: the per-block gathers / reductions carry host-side epochs and events)
        self.use_graph = bool(kernels.get("cuda_graph", True)) and zero3 is None
        self._graphs: dict[tuple, Any] = {}
        if self.attn_mode == "b200" and cfg.d_head not in (64, 128):
            # the wgmma attention kernels cover d_head 64 and 128 (every shipped MPT config); anything else uses the
            # library attention for BOTH directions (explicit + logged; GEMM/LN/CE/optimizer stay on our kernels)
            print(f"[engine] d_head={cfg.d_head}: attention falls back to SDPA (wgmma kernels cover d_head 64 / 128)", flush=True)
            self.attn_mode = "torch"
        self.model = MPTForCausalLM(cfg, device=self.device, seed=seed)
        self.frozen = apply_freeze(self.model, frozen_layers, unfrozen_layers)
        if zero3 is not None:
            from photon_b200.parallel.zero3 import ShardedFlat

            # same initial weights as an unsharded engine with this seed: materialise once, keep the shard, drop the rest
            init = FlatParams(self.model, device=self.device, with_grad=False)
            if init.layout.total != zero3.plan.layout.total or init.layout.names != zero3.plan.layout.names:
                raise ValueError("the ZeRO-3 communicator was planned for a different parameter layout")
            zero3.load_full_params(init.params)
            del init
            self.model = None
            self.flat = ShardedFlat(zero3)
            self.bf16_params = zero3.w16        # this rank's shard of the bf16 weights (what the optimizer kernel writes)
        else:
            self.flat = FlatParams(self.model, device=self.device, params_storage=params_storage, grads_storage=grads_storage)
            # bf16 compute copy; lives in a symmetric arena plane when a fused NVLink step writes it from peer GPUs
            self.bf16_params = shadow_storage if shadow_storage is not None else torch.zeros(
                self.flat.layout.total, dtype=torch.bfloat16, device=self.device)
            if self.bf16_params.numel() != self.flat.layout.total or self.bf16_params.dtype != torch.bfloat16:
                raise ValueError("shadow_storage must be a bf16 tensor with layout.total elements")
        self._init_frozen_planes()
        self.plan = BackwardPlan(cfg.n_layers, self.flat.layout.names, tied=cfg.tie_word_embeddings)
        # the LM head's logit transform (logit_scale, final_logit_softcapping), applied by the fused cross-entropy kernel
        self.head_scale, self.head_cap = cfg.head_scale, cfg.final_logit_softcapping
        self.unigram_log_probs = unigram_log_probs.to(self.device) if unigram_log_probs is not None else None
        self.lm_head_chunk = int(lm_head_chunk)
        # positional variants of the MPT attention block (ref: SURVEY §5.7): ALiBi slopes enter the attention kernels,
        # RoPE rotates q / k in place after the QKV GEMM (and un-rotates their gradients)
        from photon_b200.models.mpt import alibi_slopes, rope_tables

        self.alibi = alibi_slopes(cfg.n_heads, cfg.alibi_bias_max).to(self.device, torch.float32).contiguous() if cfg.alibi else None
        self.rope = tuple(t.contiguous() for t in rope_tables(cfg.max_seq_len, cfg.d_head, cfg.rope_theta, self.device)) if cfg.rope else None
        # keep only the block inputs h[i]; every block's internals are recomputed right before its backward
        # (fsdp_config.activation_checkpointing, ref: conf/llm_config/mpt-1b.yaml:88): 16·T·d·L bytes of bf16 -> 16·T·d
        self.activation_checkpointing = bool(activation_checkpointing)
        self.collect_activation_stats = False
        self.activation_stats: dict[str, float] = {}
        self.launches_per_microbatch = 0
        self._ws: dict[tuple[int, int], dict[str, Any]] = {}
        self._stats = torch.zeros(4, dtype=torch.float64, device=self.device)
        self._bind()
        if self.fp8:
            self._init_fp8(int(kernels.get("fp8_amax_history_len", 16)), int(kernels.get("fp8_margin", 0)))
        self.params_updated()

    # ------------------------------------------------------------------ binding
    def _init_frozen_planes(self) -> None:
        """Storage of the frozen tensors (``fl.frozen_layers`` / ``fl.unfrozen_layers``): they are not in the trainable flat, so
        they get a flat layout of their own, an fp32 plane (read by LayerNorms, bias epilogues, q/k-LN) and its bf16 cast (read by
        the GEMMs). The module's frozen parameters become views of the fp32 plane, like the trainable ones of :class:`FlatParams`.
        Nothing trains them: the optimizer, the round kernels and the gradient all-reduce only see the trainable flat."""
        self.frozen_layout: FlatLayout | None = None
        self.frozen_params = self.frozen_bf16 = None
        named = sorted(((n, p) for n, p in self.model.named_parameters() if not p.requires_grad), key=lambda kv: kv[0]) \
            if self.model is not None else []
        if not named:
            return
        lay = self.frozen_layout = FlatLayout.build((n, p.shape) for n, p in named)
        self.frozen_params = torch.zeros(lay.total, dtype=torch.float32, device=self.device)
        self.frozen_bf16 = torch.zeros(lay.total, dtype=torch.bfloat16, device=self.device)
        with torch.no_grad():
            for i, (_, p) in enumerate(named):
                v = lay.view(self.frozen_params, i)
                v.copy_(p.detach())
                p.data = v

    def _bind(self) -> None:
        lay, P, G, Sd = self.flat.layout, self.flat.params, self.flat.grads, self.bf16_params
        have = set(lay.names)
        flay, FP, F16 = self.frozen_layout, self.frozen_params, self.frozen_bf16
        frozen = set(flay.names) if flay is not None else set()

        # biases are absent under `no_bias`: every consumer below accepts None (GEMM without bias, LN without beta,
        # no bias-gradient column sums); a frozen tensor is read from the frozen planes and has no gradient (None)
        def v32(n: str) -> torch.Tensor | None:
            n = "transformer." + n
            return lay.view(P, n) if n in have else flay.view(FP, n) if n in frozen else None

        def v16(n: str, pre: str = "transformer.") -> torch.Tensor:
            n = pre + n
            return flay.view(F16, n) if n in frozen else lay.view(Sd, n)

        vg = lambda n, pre="transformer.": lay.view(G, pre + n) if pre + n in have else None  # noqa: E731
        if self.zero3 is not None:
            # weights: views into the two rotating block buffers (block i -> buffer i % 2) / the resident embedding (and untied
            # head) buffers; 1-D fp32 parameters: the packed resident buffer; gradients: the unit's staging plane (reduced after
            # its backward)
            z = self.zero3
            v32 = lambda n: z.small("transformer." + n) if "transformer." + n in have else None  # noqa: E731
            vg = lambda n, pre="transformer.": z.grad(pre + n) if pre + n in have else None  # noqa: E731
            v16 = lambda n, pre="transformer.": z.weight(pre + n)  # noqa: E731
        has_wpe = self.cfg.learned_pos_emb
        self.wte16, self.wpe16 = v16("wte.weight"), (v16("wpe.weight") if has_wpe else None)
        self.d_wte, self.d_wpe = vg("wte.weight"), (vg("wpe.weight") if has_wpe else None)
        # the LM head's weight: wte when tied, else lm_head (bf16 also under amp_fp8; a frozen one reads the frozen planes)
        if self.cfg.tie_word_embeddings:
            self.head16, self.d_head16 = self.wte16, self.d_wte
        else:
            self.head16, self.d_head16 = v16("lm_head.weight", ""), vg("lm_head.weight", "")
        self.gf, self.bf, self.d_gf, self.d_bf = v32("norm_f.weight"), v32("norm_f.bias"), vg("norm_f.weight"), vg("norm_f.bias")
        self.layers: list[_LayerW] = []
        for i in range(self.cfg.n_layers):
            p = f"blocks.{i}."
            w = _LayerW()
            w.wqkv, w.wo, w.wup, w.wdown = (v16(p + "attn.Wqkv.weight"), v16(p + "attn.out_proj.weight"),
                                            v16(p + "ffn.up_proj.weight"), v16(p + "ffn.down_proj.weight"))
            w.bqkv, w.bo, w.bup, w.bdown = (v32(p + "attn.Wqkv.bias"), v32(p + "attn.out_proj.bias"),
                                            v32(p + "ffn.up_proj.bias"), v32(p + "ffn.down_proj.bias"))
            w.g1, w.b1, w.g2, w.b2 = v32(p + "norm_1.weight"), v32(p + "norm_1.bias"), v32(p + "norm_2.weight"), v32(p + "norm_2.bias")
            w.d_wqkv, w.d_wo, w.d_wup, w.d_wdown = (vg(p + "attn.Wqkv.weight"), vg(p + "attn.out_proj.weight"),
                                                    vg(p + "ffn.up_proj.weight"), vg(p + "ffn.down_proj.weight"))
            w.d_bqkv, w.d_bo, w.d_bup, w.d_bdown = (vg(p + "attn.Wqkv.bias"), vg(p + "attn.out_proj.bias"),
                                                    vg(p + "ffn.up_proj.bias"), vg(p + "ffn.down_proj.bias"))
            w.d_g1, w.d_b1, w.d_g2, w.d_b2 = vg(p + "norm_1.weight"), vg(p + "norm_1.bias"), vg(p + "norm_2.weight"), vg(p + "norm_2.bias")
            # attn_config.qk_ln: LayerNorm on the query (d_model) and key (kv_n_heads * d_head) projections
            w.qk_g = [v32(p + "attn.q_ln.weight"), v32(p + "attn.k_ln.weight")]
            w.qk_b = [v32(p + "attn.q_ln.bias"), v32(p + "attn.k_ln.bias")]
            w.d_qk_g = [vg(p + "attn.q_ln.weight"), vg(p + "attn.k_ln.weight")]
            w.d_qk_b = [vg(p + "attn.q_ln.bias"), vg(p + "attn.k_ln.bias")]
            gated = self.cfg.ffn_gated   # ffn_config.ffn_type mptglu: gate_proj next to up_proj
            w.wgate, w.bgate = (v16(p + "ffn.gate_proj.weight"), v32(p + "ffn.gate_proj.bias")) if gated else (None, None)
            w.d_wgate, w.d_bgate = (vg(p + "ffn.gate_proj.weight"), vg(p + "ffn.gate_proj.bias")) if gated else (None, None)
            self.layers.append(w)

    def params_updated(self) -> None:
        """Re-cast the bf16 compute shadow from the fp32 masters. Only needed after host-side
        parameter loads: the fused optimizer and the round-broadcast kernels write the shadow
        themselves (the Trainer skips this call in that case)."""
        if self.zero3 is not None:
            self.zero3.before_param_write()
            ops.cast_bf16(self.flat.params, self.bf16_params)
            self.zero3.params_changed()
            return
        ops.cast_bf16(self.flat.params, self.bf16_params)
        self._frozen_updated()

    def _frozen_updated(self) -> None:
        """Re-derive the frozen tensors' compute copies (bf16 cast; under amp_fp8 their E4M3 copies and weight scales) from the
        fp32 frozen plane. Training never changes that plane, so this runs only when its values are set."""
        if self.frozen_params is None:
            return
        ops.cast_bf16(self.frozen_params, self.frozen_bf16)
        if self.fp8 and self.w8f_seg is not None:
            self._fp8_quantize_frozen()

    # ---------------------------------------------------------------------- fp8
    _DYN_ROLES = ("x_ln1", "x_attn", "x_ln2", "x_u", "g_dqkv", "g_dhmid", "g_dz", "g_dh")   # per block: 4 × E4M3, 4 × E5M2
    _W_ROLES = ("wqkv", "wo", "wup", "wdown")

    def _init_fp8(self, history_len: int, margin: int) -> None:
        """Device-resident scaling state: ``meta`` = [3, n_roles] (scale, 1/scale, running amax). Roles [0, 8L) are activations
        and gradients (delayed scaling: amax history → next scale, ``ops.fp8_update_scales``); roles [8L, 12L) are the weight
        matrices (current scaling, re-quantised from the bf16 shadow at the start of every microbatch — two passes over
        ≤ 2 bytes/param, so whoever wrote the shadow (optimizer, round broadcast, ZeRO step) needs no hook).

        Frozen matrices never change: they are quantised once, whenever their values are set (:meth:`_frozen_updated`), into a
        plane at the frozen layout's offsets, with a transposed (K-major) copy next to it that their dgrad GEMMs read directly.
        Their weight roles come after the trainable ones, so each group is one contiguous role range.

        Under full parameter sharding no rank holds whole matrices: the communicator quantises them once per parameter version
        (every parameter write ends in ``params_changed``), each owner its pieces with the tensor's global amax, and gathers the
        E4M3 bytes. The weight views point into its rotating E4M3 unit buffers and the prologue re-quantises nothing."""
        L, lay, dev = self.cfg.n_layers, self.flat.layout, self.device
        self._n_dyn = len(self._DYN_ROLES) * L
        n_roles = self._n_dyn + len(self._W_ROLES) * L
        self.fp8_meta = torch.zeros(3, n_roles, dtype=torch.float32, device=dev)
        self.fp8_meta[:2] = 1.0
        self.fp8_hist = torch.zeros(self._n_dyn, max(1, history_len), dtype=torch.float32, device=dev)
        self.fp8_fmax = torch.tensor([ops.FP8_MAX[0 if j < 4 else 1] for _ in range(L) for j in range(8)], dtype=torch.float32, device=dev)
        self.fp8_pos = torch.zeros(1, dtype=torch.int32, device=dev)
        self.fp8_margin_mult = float(2.0 ** margin)
        flay, z = self.frozen_layout, self.zero3
        # E4M3 weights at the flat layout's offsets (under full sharding: the communicator's gathered units instead)
        self.w8 = torch.zeros(lay.total, dtype=torch.uint8, device=dev) if z is None else None
        self.w8f = torch.zeros(flay.total, dtype=torch.uint8, device=dev) if flay is not None else None   # ... at the frozen layout's
        seg, fseg, order, self.w8_views, self.w8t_views = [], [], [], [], []
        for i in range(L):
            for key, name in zip(self._W_ROLES, ("attn.Wqkv.weight", "attn.out_proj.weight", "ffn.up_proj.weight", "ffn.down_proj.weight")):
                n = f"transformer.blocks.{i}.{name}"
                (fseg if flay is not None and n in flay.names else seg).append((i, key, n))
            self.w8_views.append({})
            self.w8t_views.append({})
        self._w_role = {}
        for r, (i, key, n) in enumerate(seg + fseg):
            self._w_role[(i, key)] = self._n_dyn + r
        for i, key, n in seg:
            self.w8_views[i][key] = lay.view(self.w8, n) if z is None else z.weight8(n)
        for i, key, n in fseg:
            self.w8_views[i][key] = flay.view(self.w8f, n)
            N, K = flay.shapes[flay.index(n)]
            self.w8t_views[i][key] = torch.empty(K, N, dtype=torch.uint8, device=dev)   # W^T: the dgrad GEMM's K-major B operand
        table = lambda lo, s: torch.tensor([(lo.offsets[lo.index(n)], lo.numels[lo.index(n)]) for _, _, n in s],  # noqa: E731
                                           dtype=torch.int64, device=dev).reshape(-1, 2)
        self.w8f_seg = table(flay, fseg) if fseg else None
        if z is None:
            self.w8_seg = table(lay, seg)
            self._n_w8 = len(seg)
        else:
            slot = {n: j for j, n in enumerate(z.plan.weight_names)}
            roles = [0] * len(slot)
            for i, key, n in seg:
                roles[slot[n]] = self._w_role[(i, key)]
            z.attach_fp8(self.fp8_meta, roles)   # quantised from now on by every params_changed (the first one ends __init__)
            self.w8_seg, self._n_w8 = None, 0
        self._fp8_calibrated = False

    def _role(self, name: str, layer: int) -> int:
        if name in self._DYN_ROLES:
            return layer * len(self._DYN_ROLES) + self._DYN_ROLES.index(name)
        return self._w_role[(layer, name)]

    def _fp8_quantize_frozen(self) -> None:
        ops.fp8_quantize_segments(self.frozen_bf16, self.w8f, self.w8f_seg, self.fp8_meta, self._n_dyn + self._n_w8)
        for w8, w8t in zip(self.w8_views, self.w8t_views):
            for key, t in w8t.items():
                ops.transpose_u8(w8[key], t)

    def _fp8_prologue(self, train: bool) -> None:
        """Start of a microbatch: roll the delayed scales (training only) and re-quantise the trainable weights from the shadow."""
        if train:
            ops.fp8_update_scales(self.fp8_meta, self.fp8_hist, self.fp8_fmax, self.fp8_pos, self._n_dyn, self.fp8_margin_mult)
        if self._n_w8:
            ops.fp8_quantize_segments(self.bf16_params, self.w8, self.w8_seg, self.fp8_meta, self._n_dyn)

    def fp8_state_dict(self) -> dict[str, Any] | None:
        """Scales / amax histories, checkpointed next to the optimizer so a resumed run casts with the scales it stopped with."""
        if not self.fp8:
            return None
        return {"meta": self.fp8_meta.cpu(), "hist": self.fp8_hist.cpu(), "pos": self.fp8_pos.cpu(), "calibrated": self._fp8_calibrated}

    def load_fp8_state_dict(self, sd: dict[str, Any]) -> None:
        if self.fp8 and sd and "meta" in sd and tuple(sd["meta"].shape) == tuple(self.fp8_meta.shape):
            self.fp8_meta.copy_(sd["meta"]), self.fp8_hist.copy_(sd["hist"]), self.fp8_pos.copy_(sd["pos"])
            self._fp8_calibrated = bool(sd.get("calibrated", True))
            if self.w8f_seg is not None:   # the frozen E4M3 bytes must stay paired with their (current-scaling) weight scales
                self._fp8_quantize_frozen()
            if self.zero3 is not None:     # likewise the sharded E4M3 weights (a collective: every rank loads the state)
                self.zero3.before_param_write()
                self.zero3.params_changed()

    # ---------------------------------------------------------------- workspace
    def _workspace(self, b: int, S: int) -> dict[str, Any]:
        key = (b, S)
        if key in self._ws:
            return self._ws[key]
        self._ws.clear()  # one live shape at a time (activations dominate memory)
        self._graphs.clear()  # captured graphs point into the old workspace
        c, dev = self.cfg, self.device
        T, d, H, L, W, Fh = b * S, c.d_model, c.n_heads, c.n_layers, c.qkv_dim, c.ffn_hidden
        bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
        mean = (lambda: None) if c.rmsnorm else (lambda: f32(T))   # a LayerNorm's row means (RMSNorm keeps rstd only)  # noqa: E731
        ws: dict[str, Any] = {"h": [bf(T, d) for _ in range(L + 1)], "layers": []}
        for i in range(L):
            if self.activation_checkpointing and i > 0:
                ws["layers"].append(ws["layers"][0])  # ONE set of block internals shared by all layers
                continue
            if self.fp8:   # the GEMM inputs exist only as E4M3 (1 byte): 7·T·d instead of 12·T·d bytes of saved activations
                u8 = lambda *s: torch.empty(*s, dtype=torch.uint8, device=dev)  # noqa: E731
                ws["layers"].append({"ln1": u8(T, d), "m1": mean(), "r1": f32(T), "qkv": bf(T, W), "attn": bf(T, d), "attn8": u8(T, d),
                                     "lse": f32(b, H, S), "hmid": bf(T, d), "ln2": u8(T, d), "m2": mean(), "r2": f32(T),
                                     "z": bf(T, Fh), "u": u8(T, Fh)})
            else:
                ws["layers"].append({"ln1": bf(T, d), "m1": mean(), "r1": f32(T), "qkv": bf(T, W), "attn": bf(T, d),
                                     "lse": f32(b, H, S), "hmid": bf(T, d), "ln2": bf(T, d), "m2": mean(), "r2": f32(T),
                                     "z": bf(T, Fh), "u": bf(T, Fh)})
                if c.ffn_gated:   # z = u * act'(g), u = act(g) * up (the down projection's input), a = act(g)
                    ws["layers"][-1]["a"] = bf(T, Fh)
            if c.clip_qkv:
                ws["layers"][-1]["clipmask"] = torch.empty(T, W, dtype=torch.bool, device=dev)
            if c.qk_ln:   # pre-norm q / k (inputs of the two norm backward passes) and their row statistics
                ws["layers"][-1].update(qk_pre=[bf(T, d), bf(T, c.kv_dim)], qk_m=[mean(), mean()], qk_r=[f32(T), f32(T)])
        if c.qk_ln:   # scratch of the q / k norms, viewed at the width of the part in use (see _qk_parts)
            ws.update(qk_tmp=bf(T, d), qk_tmp2=bf(T, d))
        ws.update(lnf=bf(T, d), mf=mean(), rf=f32(T), dlnf=bf(T, d), dh=bf(T, d), dhmid=bf(T, d), dln=bf(T, d),
                  dqkv=bf(T, W), dattn=bf(T, d), dz=bf(T, Fh), delta=f32(b, H, S),
                  logits=bf(min(self.lm_head_chunk, T), c.vocab_size))
        if self.fp8:   # E5M2 copy of the gradient currently flowing backward (one buffer, viewed at the width in use)
            ws["g8"] = torch.empty(T * max(Fh, 3 * d), dtype=torch.uint8, device=dev)
        if c.attn_uses_sequence_id:   # first / last row of each row's document, shared by every layer and both directions
            ws.update(doc_start=torch.empty(T, dtype=torch.int32, device=dev), doc_end=torch.empty(T, dtype=torch.int32, device=dev))
        if c.ffn_gated:   # the gate's output gradient (the up projection's goes to dz)
            ws["dg"] = bf(T, Fh)
        ws["sequence_id"] = None      # this microbatch's document ids (set by _forward), None: plain causal
        self._ws[key] = ws
        return ws

    # ------------------------------------------------------------ normalisation
    # Every norm of the model (norm_1, norm_2, norm_f, q_ln, k_ln) runs through these three, LayerNorm or RMSNorm by
    # cfg.norm_type. ``b`` (beta), ``db`` and ``m`` (row means) belong to LayerNorm only: RMSNorm ignores them (None there).
    def _norm_fwd(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor | None, y: torch.Tensor, m: torch.Tensor | None,
                  r: torch.Tensor) -> None:
        if self.cfg.rmsnorm:
            ops.rmsnorm_fwd(x, g, y, r, self.cfg.norm_eps)
        else:
            ops.layernorm_fwd(x, g, b, y, m, r, self.cfg.norm_eps)

    def _norm_fwd_q8(self, x: torch.Tensor, g: torch.Tensor, b: torch.Tensor | None, y8: torch.Tensor, m: torch.Tensor | None,
                     r: torch.Tensor, role: int) -> None:
        if self.cfg.rmsnorm:
            ops.rmsnorm_fwd_q8(x, g, y8, r, self.cfg.norm_eps, self.fp8_meta, role)
        else:
            ops.layernorm_fwd_q8(x, g, b, y8, m, r, self.cfg.norm_eps, self.fp8_meta, role)

    def _norm_bwd(self, dy: torch.Tensor, x: torch.Tensor, g: torch.Tensor, m: torch.Tensor | None, r: torch.Tensor,
                  dres: torch.Tensor | None, dx: torch.Tensor, dg: torch.Tensor | None, db: torch.Tensor | None) -> None:
        if self.cfg.rmsnorm:
            ops.rmsnorm_bwd(dy, x, g, r, dres, dx, dg)
        else:
            ops.layernorm_bwd(dy, x, g, m, r, dres, dx, dg, db)

    # ------------------------------------------------------------------ forward
    def _kernel_attention(self, S: int) -> bool:
        return self.attn_mode == "b200" and S % 128 == 0

    def _qk_parts(self) -> tuple[tuple[int, int], tuple[int, int]]:
        """(first column, width) of q and of k in a fused qkv row: what ``q_ln`` / ``k_ln`` normalise."""
        c = self.cfg
        return (0, c.d_model), (c.d_model, c.kv_dim)

    def _sdpa_heads(self, qkv: torch.Tensor, b: int, S: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
        """q [b, H, S, dh] and k, v [b, H_kv, S, dh]: views of the fused qkv."""
        c = self.cfg
        x = qkv.view(b, S, c.qkv_dim)
        d, kvd = c.d_model, c.kv_dim
        q = x[..., :d].view(b, S, c.n_heads, c.d_head).transpose(1, 2)
        k, v = (x[..., lo:lo + kvd].view(b, S, c.kv_n_heads, c.d_head).transpose(1, 2) for lo in (d, d + kvd))
        return q, k, v

    def _attention_fwd(self, lw: dict[str, Any], ws: dict[str, Any], b: int, S: int) -> None:
        c = self.cfg
        scale = c.attn_scale
        doc = ws["sequence_id"] is not None
        if self._kernel_attention(S):
            ops.attention_fwd(lw["qkv"].view(b, S, c.qkv_dim), lw["attn"].view(b, S, c.d_model), lw["lse"], c.n_heads, scale, True,
                              self.alibi, ws["doc_start"] if doc else None, n_kv_heads=c.kv_n_heads, window=c.sliding_window_size)
            return
        # library attention: kernels.attention=torch, an unsupported d_head, or a sequence length that is not a multiple
        # of the 128-row tiles (the shipped configs use 2048)
        q, k, v = self._sdpa_heads(lw["qkv"], b, S)
        o = F.scaled_dot_product_attention(q, k, v, scale=scale, **self._sdpa_mask(S, q.dtype, ws["sequence_id"]), **self._gqa())
        lw["attn"].view(b, S, c.n_heads, c.d_head).copy_(o.transpose(1, 2))

    def _gqa(self) -> dict[str, Any]:
        return {"enable_gqa": True} if self.cfg.kv_n_heads != self.cfg.n_heads else {}

    def _sdpa_mask(self, S: int, dtype: torch.dtype, sequence_id: torch.Tensor | None = None) -> dict[str, Any]:
        win = window_keep(S, self.cfg.sliding_window_size, self.device)
        if self.alibi is None and sequence_id is None and win is None:
            return {"is_causal": True}
        keep = torch.ones(S, S, dtype=torch.bool, device=self.device).tril()
        if sequence_id is not None:   # the same equality mask as the torch module: [b, 1, S, S]
            keep = keep & (sequence_id[:, :, None] == sequence_id[:, None, :])[:, None]
        if win is not None:
            keep = keep & win
        if self.alibi is None:
            return {"attn_mask": keep}
        pos = torch.arange(S, device=self.device)
        bias = self.alibi[:, None, None] * (pos[None, :] - pos[:, None]).clamp(max=0).float()[None]
        return {"attn_mask": bias[None].masked_fill(~keep, float("-inf")).to(dtype)}

    def _attention_bwd(self, lw: dict[str, Any], ws: dict[str, Any], b: int, S: int) -> None:
        c = self.cfg
        scale = c.attn_scale
        doc = ws["sequence_id"] is not None
        if self._kernel_attention(S):
            ops.attention_bwd(lw["qkv"].view(b, S, c.qkv_dim), lw["attn"].view(b, S, c.d_model),
                              ws["dattn"].view(b, S, c.d_model), lw["lse"], ws["dqkv"].view(b, S, c.qkv_dim), ws["delta"],
                              c.n_heads, scale, True, self.alibi, ws["doc_start"] if doc else None, ws["doc_end"] if doc else None,
                              n_kv_heads=c.kv_n_heads, window=c.sliding_window_size)
            if self.rope is not None:   # gradients w.r.t. the un-rotated q, k
                ops.rope_(ws["dqkv"].view(b, S, c.qkv_dim), self.rope[0], self.rope[1], c.n_heads, inverse=True, n_kv_heads=c.kv_n_heads)
            return
        with torch.enable_grad():
            qkv = lw["qkv"].view(b, S, c.qkv_dim).detach().requires_grad_(True)
            q, k, v = self._sdpa_heads(qkv, b, S)
            o = F.scaled_dot_product_attention(q, k, v, scale=scale, **self._sdpa_mask(S, q.dtype, ws["sequence_id"]), **self._gqa())
            (g,) = torch.autograd.grad(o, qkv, ws["dattn"].view(b, S, c.n_heads, c.d_head).transpose(1, 2))
        ws["dqkv"].view(b, S, c.qkv_dim).copy_(g)
        if self.rope is not None:
            ops.rope_(ws["dqkv"].view(b, S, c.qkv_dim), self.rope[0], self.rope[1], c.n_heads, inverse=True, n_kv_heads=c.kv_n_heads)

    def _block_fwd(self, i: int, ws: dict[str, Any], b: int, S: int) -> None:
        """h[i] -> h[i+1]; the block internals land in ws["layers"][i] (also the recompute step under checkpointing)."""
        c, h, w, lw = self.cfg, ws["h"], self.layers[i], ws["layers"][i]
        if self.fp8:
            M, w8, R = self.fp8_meta, self.w8_views[i], self._role
            self._norm_fwd_q8(h[i], w.g1, w.b1, lw["ln1"], lw["m1"], lw["r1"], R("x_ln1", i))
            ops.gemm_fp8(lw["ln1"], w8["wqkv"], lw["qkv"], M, R("x_ln1", i), R("wqkv", i), bias=w.bqkv)
        else:
            self._norm_fwd(h[i], w.g1, w.b1, lw["ln1"], lw["m1"], lw["r1"])
            ops.linear_fwd(lw["ln1"], w.wqkv, w.bqkv, lw["qkv"])
        if c.clip_qkv:   # attn_config.clip_qkv: clamp the fused projection; remember where the gradient passes (inside the
            # clip or exactly on it, as torch.clamp's backward: a bf16 value lands on ±clip often)
            torch.logical_and(lw["qkv"] >= -c.clip_qkv, lw["qkv"] <= c.clip_qkv, out=lw["clipmask"])
            lw["qkv"].clamp_(-c.clip_qkv, c.clip_qkv)
        if c.qk_ln:   # q / k are strided inside the fused buffer: normalise contiguous copies
            T = lw["qkv"].shape[0]
            for j, (lo, n) in enumerate(self._qk_parts()):
                part, tmp = lw["qkv"][:, lo:lo + n], ws["qk_tmp"].view(-1)[: T * n].view(T, n)
                lw["qk_pre"][j].copy_(part)
                self._norm_fwd(lw["qk_pre"][j], w.qk_g[j], w.qk_b[j], tmp, lw["qk_m"][j], lw["qk_r"][j])
                part.copy_(tmp)
        if self.rope is not None:
            ops.rope_(lw["qkv"].view(b, S, c.qkv_dim), self.rope[0], self.rope[1], c.n_heads, n_kv_heads=c.kv_n_heads)
        self._attention_fwd(lw, ws, b, S)
        if self.fp8:
            ops.colsum_quant(lw["attn"], None, lw["attn8"], ops.E4M3, M, R("x_attn", i))
            ops.gemm_fp8(lw["attn8"], w8["wo"], lw["hmid"], M, R("x_attn", i), R("wo", i), epi=ops.EPI_RESIDUAL, bias=w.bo, aux=h[i])
            self._norm_fwd_q8(lw["hmid"], w.g2, w.b2, lw["ln2"], lw["m2"], lw["r2"], R("x_ln2", i))
            # gelu(z) leaves the epilogue as E4M3 (the down-projection's operand), gelu'(z) as bf16 (the dgrad multiplier)
            ops.gemm_fp8(lw["ln2"], w8["wup"], lw["z"], M, R("x_ln2", i), R("wup", i), epi=ops.EPI_GELU_GRAD_Q8, bias=w.bup, out2=lw["z"],
                         out8=lw["u"], role_out=R("x_u", i))
            ops.gemm_fp8(lw["u"], w8["wdown"], h[i + 1], M, R("x_u", i), R("wdown", i), epi=ops.EPI_RESIDUAL, bias=w.bdown, aux=lw["hmid"])
            return
        ops.linear_fwd(lw["attn"], w.wo, w.bo, lw["hmid"], residual=h[i])
        self._norm_fwd(lw["hmid"], w.g2, w.b2, lw["ln2"], lw["m2"], lw["r2"])
        if c.ffn_gated:
            # a = act(g), act'(g) into the free dz (a backward buffer); then u = up(ln2): lw["u"] = a * u, lw["z"] = u * act'(g)
            ops.linear_act_grad_fwd(c.ffn_act, lw["ln2"], w.wgate, w.bgate, ws["dz"], lw["a"])
            ops.linear_glu_up_fwd(lw["ln2"], w.wup, w.bup, lw["a"], ws["dz"], lw["u"], lw["z"])
        else:
            ops.linear_act_grad_fwd(c.ffn_act, lw["ln2"], w.wup, w.bup, lw["z"], lw["u"])   # lw["z"] holds act'(pre-activation)
        ops.linear_fwd(lw["u"], w.wdown, w.bdown, h[i + 1], residual=lw["hmid"])

    def _forward(self, ids: torch.Tensor, ws: dict[str, Any], sequence_id: torch.Tensor | None = None) -> None:
        """``sequence_id``: document ids of the rows (already checked by :func:`check_sequence_id`), None: plain causal. The
        kernels' document bounds are computed once here for every layer, the backward and its recompute."""
        c = self.cfg
        b, S = ids.shape
        h = ws["h"]
        z = self.zero3
        ws["sequence_id"] = sequence_id
        if sequence_id is not None and self._kernel_attention(S):
            ops.doc_bounds(sequence_id, ws["doc_start"], ws["doc_end"])
        if z is not None:
            z.ensure_resident()
        ops.embed_fwd(ids.reshape(-1), self.wte16, self.wpe16, h[0], S)
        for i in range(c.n_layers):
            if z is not None:
                z.acquire(i)          # block i's weights are in buffer i % 2 (stream-ordered wait) ...
                z.prefetch(i + 1)     # ... and block i+1 streams into the other one while block i computes
            self._block_fwd(i, ws, b, S)
            if self.collect_activation_stats:
                x = h[i + 1][:S].float()
                self.activation_stats[f"l2_norm/block_{i}"] = float(x.norm(dim=-1).mean())
                self.activation_stats[f"max/block_{i}"] = float(x.abs().max())
        self._norm_fwd(h[c.n_layers], self.gf, self.bf, ws["lnf"], ws["mf"], ws["rf"])

    def _head(self, ws: dict[str, Any], targets: torch.Tensor, grad_scale: float, train: bool) -> None:
        """Chunked LM head + fused CE (+ immediate head backward when training)."""
        T = targets.numel()
        step = ws["logits"].shape[0]
        for lo in range(0, T, step):
            hi = min(T, lo + step)
            logits = ws["logits"][: hi - lo]
            ops.gemm(ws["lnf"][lo:hi], self.head16, logits)
            ops.cross_entropy(logits, targets[lo:hi], grad_scale, train, self._stats, None, self.unigram_log_probs, self.head_scale,
                              self.head_cap)
            if train:
                if self.plan.dx("head"):
                    ops.linear_dgrad(logits, self.head16, ws["dlnf"][lo:hi])
                if self.plan.head_wgrad:   # accumulates over the chunks into wte's or lm_head's gradient
                    ops.linear_wgrad(logits, ws["lnf"][lo:hi], self.d_head16, accumulate=True)

    # ----------------------------------------------------------------- backward
    def _linear_bwd(self, i: int, ws: dict[str, Any], dy: torch.Tensor, g_role: str, x: torch.Tensor, x_role: str, w_role: str,
                    w16: torch.Tensor, dw: torch.Tensor | None, db: torch.Tensor | None, dx: torch.Tensor | None,
                    mul: torch.Tensor | None = None) -> None:
        """Backward of ``y = x @ w^T + b``: db += colsum(dy); dw += dy^T x; dx = dy w (optionally ``* mul``). A None ``dw`` /
        ``db`` / ``dx`` (frozen weight / bias, no trainable tensor below) skips that GEMM or column sum.
        fp8: the column-sum pass also emits the E5M2 copy of ``dy`` both GEMMs read; ``x`` is the saved E4M3 input."""
        if not self.fp8:
            if db is not None:
                ops.col_sum(dy, db)
            if dw is not None:
                ops.linear_wgrad(dy, x, dw)
            if dx is not None:
                ops.linear_dgrad(dy, w16, dx, mul=mul)
            return
        M, R = self.fp8_meta, self._role
        T, n = dy.shape
        dy8 = ws["g8"][: T * n].view(T, n) if dw is not None or dx is not None else None
        if dy8 is not None or db is not None:
            ops.colsum_quant(dy, db, dy8, ops.E5M2, M, R(g_role, i))
        if dw is not None:
            ops.gemm_fp8(dy8, x, dw, M, R(g_role, i), R(x_role, i), a_mn=True, b_mn=True, epi=ops.EPI_F32, a_fmt=ops.E5M2,
                         b_fmt=ops.E4M3, accumulate=True)
        if dx is not None:
            # a frozen weight has a resident K-major (transposed) copy; a trainable one is transposed by the GEMM binding
            wt = self.w8t_views[i].get(w_role)
            ops.gemm_fp8(dy8, wt if wt is not None else self.w8_views[i][w_role], dx, M, R(g_role, i), R(w_role, i), b_mn=wt is None,
                         epi=ops.EPI_MUL if mul is not None else ops.EPI_BF16, a_fmt=ops.E5M2, b_fmt=ops.E4M3, aux=mul)

    def _glu_bwd(self, i: int, ws: dict[str, Any], d_in: bool, dln: torch.Tensor | None) -> None:
        """Gated FFN backward (bf16): down's weight / bias gradients and, when ``d_in``, du = (dh W_down) * act(g) and
        dg = (dh W_down) * c in one dgrad; then the up and gate projections' trainable gradients and, when ``dln`` is given,
        dln = dg W_gate + du W_up (two dgrads, the second adding the first through its residual epilogue)."""
        w, lw, dh = self.layers[i], ws["layers"][i], ws["dh"]
        self._linear_bwd(i, ws, dh, "g_dh", lw["u"], "x_u", "wdown", w.wdown, w.d_wdown, w.d_bdown, None)
        if not d_in:
            return
        du, dg = ws["dz"], ws["dg"]
        ops.linear_glu_dgrad(dh, w.wdown, lw["a"], lw["z"], du, dg)
        self._linear_bwd(i, ws, du, "g_dz", lw["ln2"], "x_ln2", "wup", w.wup, w.d_wup, w.d_bup, None)
        self._linear_bwd(i, ws, dg, "g_dz", lw["ln2"], "x_ln2", "wgate", w.wgate, w.d_wgate, w.d_bgate, None)
        if dln is not None:
            ops.linear_dgrad(dg, w.wgate, ws["dattn"])   # dattn is free until the out-projection's dgrad writes it
            ops.linear_dgrad(du, w.wup, dln, residual=ws["dattn"])

    def _backward(self, ids: torch.Tensor, ws: dict[str, Any]) -> None:
        c = self.cfg
        b, S = ids.shape
        h = ws["h"]
        dh = ws["dh"]
        z, P = self.zero3, self.plan
        if P.runs("norm_f"):
            self._norm_bwd(ws["dlnf"], h[c.n_layers], self.gf, ws["mf"], ws["rf"], None, dh, self.d_gf, self.d_bf)
        # blocks below the lowest one with a trainable tensor (and their recompute) are skipped: see BackwardPlan
        for i in range(c.n_layers - 1, P.lowest_block - 1, -1):
            if z is not None:
                z.acquire(i)
                z.prefetch(i - 1)
                z.zero_stage(i)       # this microbatch's gradient of block i (the shard accumulates over microbatches)
            if self.activation_checkpointing and i < c.n_layers - 1:
                self._block_fwd(i, ws, b, S)   # recompute (the shared buffers still hold the LAST block after the forward)
            self._block_bwd(i, ws, b, S)
            if z is not None:
                z.reduce(i)           # reduce-scatter: every rank adds the mean of ITS slice into its gradient shard
        if P.runs("embed"):
            ops.embed_bwd(ids.reshape(-1), dh, self.d_wte, self.d_wpe, S)
        if z is not None:
            z.reduce(z.plan.rest)

    def _block_bwd(self, i: int, ws: dict[str, Any], b: int, S: int) -> None:
        """dh (gradient w.r.t. h[i+1]) -> dh (w.r.t. h[i]), accumulating block i's trainable parameter gradients; returns after the
        last stage the plan runs (the lowest trainable block only)."""
        c, h, w, lw, P = self.cfg, ws["h"], self.layers[i], ws["layers"][i], self.plan
        dh, dhmid, dln = ws["dh"], ws["dhmid"], ws["dln"]
        dx = lambda s, t: t if P.dx((i, s)) else None  # noqa: E731
        # ---- FFN: h[i+1] = hmid + down(act(up(ln2(hmid))))  or, gated, hmid + down(act(gate(ln2)) * up(ln2))
        if c.ffn_gated:
            self._glu_bwd(i, ws, P.dx((i, "down")), dx("up", dln))
        else:
            self._linear_bwd(i, ws, dh, "g_dh", lw["u"], "x_u", "wdown", w.wdown, w.d_wdown, w.d_bdown, dx("down", ws["dz"]), mul=lw["z"])
            if not P.runs((i, "up")):
                return
            self._linear_bwd(i, ws, ws["dz"], "g_dz", lw["ln2"], "x_ln2", "wup", w.wup, w.d_wup, w.d_bup, dx("up", dln))
        if not P.runs((i, "ln2")):
            return
        self._norm_bwd(dln, lw["hmid"], w.g2, lw["m2"], lw["r2"], dh, dhmid, w.d_g2, w.d_b2)
        if not P.runs((i, "out")):
            return
        # ---- attention: hmid = h[i] + out_proj(attn(qkv(ln1(h[i]))))
        self._linear_bwd(i, ws, dhmid, "g_dhmid", lw["attn8"] if self.fp8 else lw["attn"], "x_attn", "wo", w.wo, w.d_wo, w.d_bo,
                         dx("out", ws["dattn"]))
        if not P.runs((i, "attn")):
            return
        self._attention_bwd(lw, ws, b, S)
        if c.qk_ln:
            T = ws["dqkv"].shape[0]
            for j, (lo, n) in enumerate(self._qk_parts()):
                part = ws["dqkv"][:, lo:lo + n]
                tmp, tmp2 = (ws[k].view(-1)[: T * n].view(T, n) for k in ("qk_tmp", "qk_tmp2"))
                tmp.copy_(part)
                self._norm_bwd(tmp, lw["qk_pre"][j], w.qk_g[j], lw["qk_m"][j], lw["qk_r"][j], None, tmp2, w.d_qk_g[j], w.d_qk_b[j])
                part.copy_(tmp2)
        if c.clip_qkv:
            ws["dqkv"].mul_(lw["clipmask"])
        if not P.runs((i, "qkv")):
            return
        self._linear_bwd(i, ws, ws["dqkv"], "g_dqkv", lw["ln1"], "x_ln1", "wqkv", w.wqkv, w.d_wqkv, w.d_bqkv, dx("qkv", dln))
        if not P.runs((i, "ln1")):
            return
        self._norm_bwd(dln, h[i], w.g1, lw["m1"], lw["r1"], dhmid, dh, w.d_g1, w.d_b1)

    # ---------------------------------------------------------------- protocol
    def _fwd_bwd_eager(self, ids: torch.Tensor, grad_scale: float, sequence_id: torch.Tensor | None = None) -> None:
        b, S = ids.shape
        ws = self._workspace(b, S)
        targets = shift_labels(ids).reshape(-1)
        self._stats.zero_()
        if self.fp8:
            self._fp8_prologue(train=True)
        z = self.zero3
        if z is not None:
            z.zero_stage(z.plan.rest)     # embeddings + final norm collect gradients over the whole backward
            if z.plan.head is not None:
                z.zero_stage(z.plan.head)     # the untied LM head's gradient of this microbatch
        self._forward(ids, ws, sequence_id)
        self._head(ws, targets, grad_scale, train=True)
        if z is not None and z.plan.head is not None:
            z.reduce(z.plan.head)         # complete after the head's wgrad over every chunk
        self._backward(ids, ws)

    def fwd_bwd(self, ids: torch.Tensor, denom: float, scale: float = 1.0,
                sequence_id: torch.Tensor | None = None) -> tuple[torch.Tensor, torch.Tensor]:
        """Accumulate d(Σ token-loss · scale / denom) into ``flat.grads``; returns (loss_sum, n_tokens). ``sequence_id`` [b, S]
        (int64, ids non-decreasing along each row): document ids, applied when ``attn_uses_sequence_id`` is on."""
        b, S = ids.shape
        sequence_id = check_sequence_id(self.cfg, sequence_id, train=True)
        if sequence_id is not None:
            sequence_id = sequence_id.to(self.device, torch.int64, non_blocking=True).contiguous()
        grad_scale = scale / denom
        if self.fp8 and not self._fp8_calibrated:
            # delayed scaling has no history yet: one discarded pass at scale 1 records every role's amax (gradients would
            # underflow E5M2 unscaled), the next prologue turns them into scales
            saved = self.flat.grads.clone()
            self._fwd_bwd_eager(ids, grad_scale, sequence_id)
            self.flat.grads.copy_(saved)
            self._fp8_calibrated = True
        graphable = self.use_graph and self.attn_mode == "b200" and S % 128 == 0 and not self.collect_activation_stats
        if not graphable:
            n0 = ops.launch_count()
            self._fwd_bwd_eager(ids, grad_scale, sequence_id)
            self.launches_per_microbatch = ops.launch_count() - n0
        else:
            # a graph with the document mask reads a static sequence_id input of its own
            key = (b, S, float(grad_scale)) if sequence_id is None else (b, S, float(grad_scale), "doc")
            g = self._graphs.get(key)
            if g is None:
                g = self._capture(ids, grad_scale, key, sequence_id)
            g["ids"].copy_(ids, non_blocking=True)
            if sequence_id is not None:
                g["sequence_id"].copy_(sequence_id, non_blocking=True)
            g["graph"].replay()
            ops.add_launch_count(self.launches_per_microbatch)   # replayed launches are still our kernels
        st = self._stats.clone()
        return st[0], st[1]

    def _capture(self, ids: torch.Tensor, grad_scale: float, key: tuple, sequence_id: torch.Tensor | None = None) -> dict[str, Any]:
        """Warm up eagerly on a side stream (lazy allocations, kernel attributes), then capture one microbatch.
        Gradients accumulate into ``flat.grads`` — they are saved around the warm-up / capture passes."""
        if len(self._graphs) >= 4:      # shapes changed (auto microbatch, eval): drop old graphs with their static inputs
            self._graphs.clear()
        static_ids = ids.clone()
        static_sid = sequence_id.clone() if sequence_id is not None else None
        saved = self.flat.grads.clone()
        side = torch.cuda.Stream(self.device)
        side.wait_stream(torch.cuda.current_stream(self.device))
        with torch.cuda.stream(side):
            n0 = ops.launch_count()
            self._fwd_bwd_eager(static_ids, grad_scale, static_sid)
            self.launches_per_microbatch = ops.launch_count() - n0
        torch.cuda.current_stream(self.device).wait_stream(side)
        graph = torch.cuda.CUDAGraph()
        with torch.cuda.graph(graph):
            self._fwd_bwd_eager(static_ids, grad_scale, static_sid)
        self.flat.grads.copy_(saved)
        g = {"graph": graph, "ids": static_ids, "sequence_id": static_sid}
        self._graphs[key] = g
        return g

    @torch.no_grad()
    def eval_stats(self, ids: torch.Tensor, sequence_id: torch.Tensor | None = None) -> dict[str, torch.Tensor]:
        b, S = ids.shape
        sequence_id = check_sequence_id(self.cfg, sequence_id, train=False)
        if sequence_id is not None:
            sequence_id = sequence_id.to(self.device, torch.int64).contiguous()
        ws = self._workspace(b, S)
        targets = shift_labels(ids).reshape(-1)
        self._stats.zero_()
        if self.fp8:
            # evaluation casts with the training scales and leaves the delayed-scaling state as it found it: the amax its
            # forward records would otherwise be merged into the next training step's history slot, so how often a run
            # evaluates would change its training scales
            amax = self.fp8_meta[2, : self._n_dyn].clone()
            self._fp8_prologue(train=False)
        self._forward(ids, ws, sequence_id)
        if self.fp8:
            self.fp8_meta[2, : self._n_dyn].copy_(amax)
        self._head(ws, targets, 0.0, train=False)
        st = self._stats.clone()
        out = {"loss_sum": st[0], "n_tokens": st[1], "n_correct": st[2]}
        if self.unigram_log_probs is not None:
            out["unigram_loss_sum"] = st[3]
        return out

    @torch.no_grad()
    def logits(self, ids: torch.Tensor) -> torch.Tensor:
        """``[B,S] → [B,S,V]`` for the in-context-learning evaluator. ICL prompts are ragged single sequences scored a
        handful of tokens at a time — nothing like the fixed ``[b, 2048]`` schedule the kernel workspace is laid out for — so
        this runs the torch module that shares the fp32 master weights (bf16 autocast, SDPA); it is an evaluation utility,
        not part of the training step."""
        if self.model is None:
            # full parameter sharding: the evaluation utility gets a temporary whole-model copy, pulled from the owners by THIS rank's
            # copy engines (peers only have to leave their shards alone — the trainer keeps them at a barrier during the ICL suite);
            # it is rebuilt when the parameters have changed and dropped by ``train_mode(True)``
            ver = self.zero3.version
            if getattr(self, "_eval_model", None) is None or self._eval_model_version != ver:
                m = MPTForCausalLM(self.cfg, device=self.device, seed=0)
                fp = FlatParams(m, device=self.device, with_grad=False)
                fp.params.copy_(self.flat.full_params())
                m.train(False)
                self._eval_model, self._eval_model_version = m, ver
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return self._eval_model(ids.to(self.device))
        with torch.autocast("cuda", dtype=torch.bfloat16):
            return self.model(ids.to(self.device))

    def decoder(self, max_batch: int) -> Any:
        """A KV-cached greedy decoder (:class:`photon_b200.models.decode.KVDecoder`) over this engine's bf16 weights for batches of
        up to ``max_batch`` sequences, or None where it does not apply: full parameter sharding, a d_head the wgmma attention
        kernels do not cover, or a ``max_seq_len`` that is not a multiple of the 128-row prefill tiles. It owns its cache and
        buffers; the training workspace and captured training graphs are left alone."""
        if self.zero3 is not None or self.cfg.d_head not in (64, 128) or self.cfg.max_seq_len % 128:
            return None
        from photon_b200.models.decode import KVDecoder

        return KVDecoder(self, max_batch, use_graph=self.use_graph)

    def train_mode(self, on: bool = True) -> None:
        if self.model is not None:
            self.model.train(on)
        elif on:
            self._eval_model = None       # the whole-model evaluation copy (full sharding) does not outlive the evaluation

    def close(self) -> None:
        self._graphs.clear()
        self._ws.clear()
