"""KV-cached greedy decoding on the sm_90a engine (:meth:`B200Engine.decoder`).

Prefill runs the prompts of a batch, right-padded to a multiple of 128, through the training kernels (LayerNorm, wgmma GEMM,
flash attention, RoPE); after each block's attention the layer's k / v of the prompt positions go into the cache. Under causal
attention right padding never reaches a valid row, so the padded batch is exact for every prompt. Each decode step then
processes one new token per sequence:

    embed (per-row position) -> per block: LN -> QKV -> (clip / qk_ln) -> append (RoPE + cache write) -> decode attention
    -> out-proj + residual -> LN -> up + GELU -> down + residual -> final LN -> LM head -> argmax (on the device)

The step is captured as one CUDA graph per batch size and replayed; token ids, positions and the cache are static device
buffers, and the host reads back one int32 per sequence. The GEMMs of a step use the weight-streaming skinny GEMM up to
``SKINNY_MAX_M`` rows and the training GEMM above.

Cache layout: bf16 ``[L, 2, B, H, max_seq_len, d_head]`` (k = index 0, v = 1), see ``csrc/decode.h``. It is allocated for the
largest batch the decoder has been asked to run (at most ``max_batch``). The weights are the engine's bf16 compute shadow,
also under ``amp_fp8``; the decoder never touches the training workspace or its captured graphs.
"""
from __future__ import annotations

import math
from typing import Any

import torch

from photon_b200 import ops

# Up to this many rows a step's GEMMs run on the skinny (weight-streaming) GEMM, above it on the training GEMM; the
# skinny kernel covers M <= 64. Measured crossover: docs/KERNELS.md ("Decoding").
SKINNY_MAX_M = 64


class KVDecoder:
    """Batched greedy decoder over an engine's weights. ``start(prompts, max_new_tokens)`` prefills and returns the first new
    token of every row; each ``step()`` returns the next one."""

    def __init__(self, engine: Any, max_batch: int, use_graph: bool = True) -> None:
        c = engine.cfg
        if int(max_batch) < 1:
            raise ValueError("max_batch must be >= 1")
        self.e, self.cfg = engine, c
        self.max_batch, self.max_seq_len = int(max_batch), int(c.max_seq_len)
        self.use_graph = bool(use_graph)
        self.dev = engine.device
        self.scale = 1.0 / math.sqrt(c.d_head)
        self._cap = 0
        self._graphs: dict[int, torch.cuda.CUDAGraph] = {}
        self._b = 0
        self._pos_host: list[int] = []

    # ------------------------------------------------------------------ buffers
    def _ensure_capacity(self, b: int) -> None:
        if b <= self._cap:
            return
        c, dev = self.cfg, self.dev
        bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
        self._graphs.clear()   # graphs point into the old buffers
        self.cache = None
        self.cache = torch.zeros(c.n_layers, 2, b, c.n_heads, self.max_seq_len, c.d_head, dtype=torch.bfloat16, device=dev)
        d, dff = c.d_model, c.expansion_ratio * c.d_model
        self.tok = torch.zeros(b, dtype=torch.int32, device=dev)
        self.pos = torch.zeros(b, dtype=torch.int32, device=dev)
        self.buf = {"h": bf(b, d), "ln": bf(b, d), "m": f32(b), "r": f32(b), "qkv": bf(b, 3 * d), "attn": bf(b, d), "hmid": bf(b, d),
                    "u": bf(b, dff), "z": bf(b, dff), "logits": bf(b, c.vocab_size)}
        if c.qk_ln:
            self.buf.update(qk_pre=bf(b, d), qk_tmp=bf(b, d))
        self._cap = b

    @property
    def logits(self) -> torch.Tensor:
        """bf16 ``[B, V]`` logits of the last prefill / step (what its argmax was taken over)."""
        return self.buf["logits"][: self._b]

    # -------------------------------------------------------------- block parts
    def _linear(self, x: torch.Tensor, w: torch.Tensor, b: torch.Tensor | None, out: torch.Tensor, residual: torch.Tensor | None = None,
                gelu: bool = False, pre: torch.Tensor | None = None) -> None:
        if x.shape[0] <= SKINNY_MAX_M:
            ops.skinny_gemm(x, w, out, b, residual, gelu)
        elif gelu:
            ops.linear_gelu_fwd(x, w, b, pre, out)
        else:
            ops.linear_fwd(x, w, b, out, residual=residual)

    def _qkv_post(self, w: Any, qkv: torch.Tensor, pre: torch.Tensor, tmp: torch.Tensor, m: torch.Tensor, r: torch.Tensor) -> None:
        """clip_qkv and qk_ln exactly as the training forward applies them."""
        c = self.cfg
        if c.clip_qkv:
            qkv.clamp_(-c.clip_qkv, c.clip_qkv)
        if c.qk_ln:
            qkv3 = qkv.view(-1, 3, c.d_model)
            for j in range(2):
                pre.copy_(qkv3[:, j])
                ops.layernorm_fwd(pre, w.qk_g[j], w.qk_b[j], tmp, m, r, c.norm_eps)
                qkv3[:, j].copy_(tmp)

    # ------------------------------------------------------------------ prefill
    @torch.no_grad()
    def start(self, prompts: list[list[int]], max_new_tokens: int) -> list[int]:
        """Prefill ``prompts`` (a batch of token lists) and return the first greedy token of each."""
        c, e = self.cfg, self.e
        b = len(prompts)
        if not 1 <= b <= self.max_batch:
            raise ValueError(f"batch of {b} prompts; this decoder runs 1..{self.max_batch}")
        lens = [len(p) for p in prompts]
        for n in lens:
            if n < 1 or n + int(max_new_tokens) > self.max_seq_len:
                raise ValueError(f"a prompt of {n} tokens plus {max_new_tokens} new tokens does not fit the {self.max_seq_len}-position cache")
        self._ensure_capacity(b)
        self._b = b
        S = -(-max(lens) // 128) * 128
        d, H, dh, T = c.d_model, c.n_heads, c.d_head, b * S
        ids = torch.zeros(b, S, dtype=torch.long)
        for i, p in enumerate(prompts):
            ids[i, : len(p)] = torch.tensor(p, dtype=torch.long)
        ids = ids.to(self.dev, non_blocking=True)
        bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=self.dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.dev)  # noqa: E731
        h, hmid, ln, qkv, attn = bf(T, d), bf(T, d), bf(T, d), bf(T, 3 * d), bf(T, d)
        m, r, lse = f32(T), f32(T), f32(b, H, S)
        u, z = bf(T, c.expansion_ratio * d), bf(T, c.expansion_ratio * d)
        pre, tmp = (bf(T, d), bf(T, d)) if c.qk_ln else (None, None)
        ops.embed_fwd(ids.reshape(-1), e.wte16, e.wpe16, h, S)
        for i, w in enumerate(e.layers):
            ops.layernorm_fwd(h, w.g1, w.b1, ln, m, r, c.norm_eps)
            ops.linear_fwd(ln, w.wqkv, w.bqkv, qkv)
            self._qkv_post(w, qkv, pre, tmp, m, r)
            if e.rope is not None:
                ops.rope_(qkv.view(b, S, 3 * d), e.rope[0], e.rope[1], H)
            ops.attention_fwd(qkv.view(b, S, 3 * d), attn.view(b, S, d), lse, H, self.scale, True, e.alibi)
            kv = qkv.view(b, S, 3, H, dh)
            self.cache[i, 0, :b, :, :S].copy_(kv[:, :, 1].transpose(1, 2))   # k / v after clip, qk_ln and RoPE
            self.cache[i, 1, :b, :, :S].copy_(kv[:, :, 2].transpose(1, 2))
            ops.linear_fwd(attn, w.wo, w.bo, hmid, residual=h)
            ops.layernorm_fwd(hmid, w.g2, w.b2, ln, m, r, c.norm_eps)
            ops.linear_gelu_fwd(ln, w.wup, w.bup, z, u)
            ops.linear_fwd(u, w.wdown, w.bdown, h, residual=hmid)
        # only the last prompt row of every sequence goes through the final LN and the LM head
        last = torch.tensor([i * S + n - 1 for i, n in enumerate(lens)], dtype=torch.long).to(self.dev, non_blocking=True)
        B = self.buf
        torch.index_select(h, 0, last, out=B["h"][:b])
        ops.layernorm_fwd(B["h"][:b], e.gf, e.bf, B["ln"][:b], B["m"][:b], B["r"][:b], c.norm_eps)
        self._linear(B["ln"][:b], e.wte16, None, B["logits"][:b])
        self.pos[:b].copy_(torch.tensor(lens, dtype=torch.int32), non_blocking=True)
        ops.argmax_advance(B["logits"][:b], self.tok[:b])
        self._pos_host = list(lens)
        return self.tok[:b].tolist()

    # --------------------------------------------------------------------- step
    def _step_kernels(self, b: int) -> None:
        c, e, B = self.cfg, self.e, self.buf
        h, ln, m, r, qkv, attn, hmid, u, z = (B[k][:b] for k in ("h", "ln", "m", "r", "qkv", "attn", "hmid", "u", "z"))
        pre, tmp = (B["qk_pre"][:b], B["qk_tmp"][:b]) if c.qk_ln else (None, None)
        ops.embed_pos(self.tok, self.pos, e.wte16, e.wpe16, h)
        for i, w in enumerate(e.layers):
            kc, vc = self.cache[i, 0], self.cache[i, 1]
            ops.layernorm_fwd(h, w.g1, w.b1, ln, m, r, c.norm_eps)
            self._linear(ln, w.wqkv, w.bqkv, qkv)
            self._qkv_post(w, qkv, pre, tmp, m, r)
            ops.decode_append(qkv, self.pos, kc, vc, e.rope, c.n_heads)
            ops.decode_attention(qkv, kc, vc, self.pos, attn, c.n_heads, self.scale, e.alibi)
            self._linear(attn, w.wo, w.bo, hmid, residual=h)
            ops.layernorm_fwd(hmid, w.g2, w.b2, ln, m, r, c.norm_eps)
            self._linear(ln, w.wup, w.bup, u, gelu=True, pre=z)
            self._linear(u, w.wdown, w.bdown, h, residual=hmid)
        ops.layernorm_fwd(h, e.gf, e.bf, ln, m, r, c.norm_eps)
        self._linear(ln, e.wte16, None, B["logits"][:b])
        ops.argmax_advance(B["logits"][:b], self.tok, self.pos)

    @torch.no_grad()
    def step(self) -> list[int]:
        """Feed the last token of every row and return the next greedy token of each."""
        b = self._b
        if b == 0:
            raise RuntimeError("start() a batch before stepping")
        if max(self._pos_host) >= self.max_seq_len:
            raise ValueError(f"a sequence reached the {self.max_seq_len}-position cache")
        if not self.use_graph:
            self._step_kernels(b)
        elif b in self._graphs:
            self._graphs[b].replay()
        else:
            self._step_kernels(b)   # the real step, eagerly: sets kernel attributes and warms the allocator for the capture
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._step_kernels(b)
            self._graphs[b] = g
        self._pos_host = [p + 1 for p in self._pos_host]
        return self.tok[:b].tolist()

    def close(self) -> None:
        self._graphs.clear()
        self.cache = None
        self.buf = {}
        self._cap = self._b = 0
