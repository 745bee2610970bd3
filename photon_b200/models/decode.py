"""KV-cached greedy decoding on the sm_90a engine (:meth:`B200Engine.decoder`).

Prefill runs the prompts of a batch, right-padded to a multiple of 128, through the training kernels (LayerNorm, wgmma GEMM,
flash attention, RoPE); after each block's attention the layer's k / v of the prompt positions go into the cache. Under causal
attention right padding never reaches a valid row, so the padded batch is exact for every prompt. Each decode step then
processes one new token per sequence:

    embed (per-row position) -> per block: LN -> QKV -> (clip / qk_ln) -> append (RoPE + cache write) -> decode attention
    -> out-proj + residual -> LN -> FFN -> down + residual -> final LN -> LM head -> argmax (on the device)

The LM head is ``wte`` or, untied, ``lm_head``. Greedy decoding takes the argmax of its raw logits: the head's transform
(``logit_scale``, ``final_logit_softcapping``) is strictly increasing, so it cannot change the argmax.

where the FFN is up + activation (GELU or SiLU) or, gated (``mptglu``), gate + activation -> up times that.

The step is captured as one CUDA graph per batch size and replayed; token ids, positions and the cache are static device
buffers, and the host reads back one int32 per sequence. The GEMMs of a step use the weight-streaming skinny GEMM up to
``SKINNY_MAX_M`` rows and the training GEMM above.

Cache layout: bf16 ``[L, 2, B, H_kv, max_seq_len, d_head]`` (k = index 0, v = 1; ``H_kv`` = ``kv_n_heads``, fewer than the query
heads with grouped-query attention), see ``csrc/decode.h``. It is allocated for the
largest batch the decoder has been asked to run (at most ``max_batch``). The weights are the engine's bf16 compute shadow,
also under ``amp_fp8``; the decoder never touches the training workspace or its captured graphs.

The same cache serves log-likelihood scoring (:meth:`KVDecoder.score`, the multiple-choice, schema and language-modelling ICL
tasks): each distinct context is prefilled once and its k / v copied into one slot per (context, continuation) pair; the
continuation tokens of every pair then run through the blocks together, several rows per slot, with cache attention (a
wgmma kernel over the slot's keys, causal at each row's own position) in place of decode attention.
"""
from __future__ import annotations

from typing import Any

import torch

from photon_b200 import ops
from photon_b200.models.mpt import head_transform

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
        self.scale, self.window = c.attn_scale, c.sliding_window_size
        self._cap = 0
        self._graphs: dict[int, torch.cuda.CUDAGraph] = {}
        self._b = 0
        self._pos_host: list[int] = []

    # ------------------------------------------------------------------ buffers
    def _ensure_capacity(self, b: int) -> None:
        if b <= self._cap:
            return
        c, dev = self.cfg, self.dev
        self._graphs.clear()   # graphs point into the old buffers
        self.cache = None
        self.cache = torch.zeros(c.n_layers, 2, b, c.kv_n_heads, self.max_seq_len, c.d_head, dtype=torch.bfloat16, device=dev)
        self.tok = torch.zeros(b, dtype=torch.int32, device=dev)
        self.pos = torch.zeros(b, dtype=torch.int32, device=dev)
        self.buf = self._row_buffers(b)
        self.buf["logits"] = torch.empty(b, c.vocab_size, dtype=torch.bfloat16, device=dev)
        self._cap = b

    def _row_buffers(self, n: int, h: torch.Tensor | None = None) -> dict[str, torch.Tensor]:
        """Activations of ``n`` rows through the blocks (``h``: the residual stream, allocated when None)."""
        c, dev = self.cfg, self.dev
        bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)  # noqa: E731
        d, dff = c.d_model, c.ffn_hidden
        x = {"h": bf(n, d) if h is None else h, "ln": bf(n, d), "m": f32(n), "r": f32(n), "qkv": bf(n, c.qkv_dim), "attn": bf(n, d),
             "hmid": bf(n, d), "u": bf(n, dff), "z": bf(n, dff)}
        if c.ffn_gated and n > SKINNY_MAX_M:   # the training GEMM's gated forward also writes act'(g) and u * act'(g)
            x.update(ffn_d=bf(n, dff), ffn_c=bf(n, dff))
        if c.qk_ln:
            x.update(qk_pre=bf(n, d), qk_tmp=bf(n, d))
        return x

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

    def _ffn(self, w: Any, ln: torch.Tensor, u: torch.Tensor, z: torch.Tensor, out: torch.Tensor, resid: torch.Tensor,
             dact: torch.Tensor | None = None, cg: torch.Tensor | None = None) -> None:
        """``out = resid + ffn(ln)``. ``u`` / ``z``: [rows, F] scratch; a gated FFN over more than ``SKINNY_MAX_M`` rows runs the
        training forward, which also writes act'(g) into ``dact`` and u * act'(g) into ``cg``."""
        c = self.cfg
        skinny = ln.shape[0] <= SKINNY_MAX_M
        if c.ffn_gated:
            if skinny:   # z = act(gate(ln)); u = up(ln) * z
                ops.skinny_gemm(ln, w.wgate, z, w.bgate, gelu=c.ffn_act == "gelu", silu=c.ffn_act == "silu")
                ops.skinny_gemm(ln, w.wup, u, w.bup, mul=z)
            else:
                ops.linear_act_grad_fwd(c.ffn_act, ln, w.wgate, w.bgate, dact, z)
                ops.linear_glu_up_fwd(ln, w.wup, w.bup, z, dact, u, cg)
        elif c.ffn_act == "silu":
            if skinny:
                ops.skinny_gemm(ln, w.wup, u, w.bup, silu=True)
            else:
                ops.linear_silu_grad_fwd(ln, w.wup, w.bup, z, u)
        else:
            self._linear(ln, w.wup, w.bup, u, gelu=True, pre=z)
        self._linear(u, w.wdown, w.bdown, out, residual=resid)

    def _qkv_post(self, w: Any, qkv: torch.Tensor, pre: torch.Tensor, tmp: torch.Tensor, m: torch.Tensor, r: torch.Tensor) -> None:
        """clip_qkv and qk_ln exactly as the training forward applies them."""
        c = self.cfg
        if c.clip_qkv:
            qkv.clamp_(-c.clip_qkv, c.clip_qkv)
        if c.qk_ln:
            T = qkv.shape[0]
            for j, (lo, n) in enumerate(self.e._qk_parts()):  # noqa: SLF001
                part = qkv[:, lo:lo + n]
                p, t = (x.view(-1)[: T * n].view(T, n) for x in (pre, tmp))
                p.copy_(part)
                self.e._norm_fwd(p, w.qk_g[j], w.qk_b[j], t, m, r)  # noqa: SLF001
                part.copy_(t)

    # ------------------------------------------------------------------ prefill
    def _prefill(self, prompts: list[list[int]], slots: list[int]) -> torch.Tensor:
        """Run ``prompts`` (right-padded to a multiple of 128) through the blocks on the training kernels, writing every layer's
        k / v of prompt ``i`` into cache slot ``slots[i]``; returns the hidden state of each prompt's last token ``[len, d]``."""
        c, e = self.cfg, self.e
        b = len(prompts)
        lens = [len(p) for p in prompts]
        S = -(-max(lens) // 128) * 128
        d, H, Hkv, dh, T, W = c.d_model, c.n_heads, c.kv_n_heads, c.d_head, b * S, c.qkv_dim
        ids = torch.zeros(b, S, dtype=torch.long)
        for i, p in enumerate(prompts):
            ids[i, : len(p)] = torch.tensor(p, dtype=torch.long)
        ids = ids.to(self.dev, non_blocking=True)
        dst = torch.tensor(slots, dtype=torch.long).to(self.dev, non_blocking=True)
        bf = lambda *s: torch.empty(*s, dtype=torch.bfloat16, device=self.dev)  # noqa: E731
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=self.dev)  # noqa: E731
        h, hmid, ln, qkv, attn = bf(T, d), bf(T, d), bf(T, d), bf(T, W), bf(T, d)
        m, r, lse = f32(T), f32(T), f32(b, H, S)
        u, z = bf(T, c.ffn_hidden), bf(T, c.ffn_hidden)
        dact, cg = (bf(T, c.ffn_hidden), bf(T, c.ffn_hidden)) if c.ffn_gated else (None, None)
        pre, tmp = (bf(T, d), bf(T, d)) if c.qk_ln else (None, None)
        ops.embed_fwd(ids.reshape(-1), e.wte16, e.wpe16, h, S)
        for i, w in enumerate(e.layers):
            e._norm_fwd(h, w.g1, w.b1, ln, m, r)
            ops.linear_fwd(ln, w.wqkv, w.bqkv, qkv)
            self._qkv_post(w, qkv, pre, tmp, m, r)
            if e.rope is not None:
                ops.rope_(qkv.view(b, S, W), e.rope[0], e.rope[1], H, n_kv_heads=Hkv)
            ops.attention_fwd(qkv.view(b, S, W), attn.view(b, S, d), lse, H, self.scale, True, e.alibi, n_kv_heads=Hkv,
                              window=self.window)
            _, k, v = e._sdpa_heads(qkv, b, S)  # noqa: SLF001
            self.cache[i, 0, :, :, :S].index_copy_(0, dst, k)   # the kv heads' k / v after clip, qk_ln and RoPE
            self.cache[i, 1, :, :, :S].index_copy_(0, dst, v)
            ops.linear_fwd(attn, w.wo, w.bo, hmid, residual=h)
            e._norm_fwd(hmid, w.g2, w.b2, ln, m, r)
            self._ffn(w, ln, u, z, h, hmid, dact, cg)
        last = torch.tensor([i * S + n - 1 for i, n in enumerate(lens)], dtype=torch.long).to(self.dev, non_blocking=True)
        return torch.index_select(h, 0, last)

    @torch.no_grad()
    def start(self, prompts: list[list[int]], max_new_tokens: int) -> list[int]:
        """Prefill ``prompts`` (a batch of token lists) and return the first greedy token of each."""
        e = self.e
        b = len(prompts)
        if not 1 <= b <= self.max_batch:
            raise ValueError(f"batch of {b} prompts; this decoder runs 1..{self.max_batch}")
        lens = [len(p) for p in prompts]
        for n in lens:
            if n < 1 or n + int(max_new_tokens) > self.max_seq_len:
                raise ValueError(f"a prompt of {n} tokens plus {max_new_tokens} new tokens does not fit the {self.max_seq_len}-position cache")
        self._ensure_capacity(b)
        self._b = b
        B = self.buf
        # only the last prompt row of every sequence goes through the final LN and the LM head
        B["h"][:b].copy_(self._prefill(prompts, list(range(b))))
        e._norm_fwd(B["h"][:b], e.gf, e.bf, B["ln"][:b], B["m"][:b], B["r"][:b])
        self._linear(B["ln"][:b], e.head16, None, B["logits"][:b])
        self.pos[:b].copy_(torch.tensor(lens, dtype=torch.int32), non_blocking=True)
        ops.argmax_advance(B["logits"][:b], self.tok[:b])
        self._pos_host = list(lens)
        return self.tok[:b].tolist()

    # --------------------------------------------------------------------- blocks over cached rows
    def _blocks(self, x: dict[str, torch.Tensor], pos: torch.Tensor, slot: torch.Tensor | None = None,
                tiles: torch.Tensor | None = None) -> None:
        """Every block over the rows of ``x`` (see ``_row_buffers``; ``h`` holds the embedded rows on entry and the last block's
        output on return). Row ``r`` sits at position ``pos[r]`` of cache slot ``slot[r]`` (slot ``r`` when None) and appends its
        k / v there. Attention is decode attention (one row per slot) or, given a ``tiles`` table, cache attention over
        several rows per slot."""
        c, e = self.cfg, self.e
        h, ln, m, r, qkv, attn, hmid, u, z = (x[k] for k in ("h", "ln", "m", "r", "qkv", "attn", "hmid", "u", "z"))
        for i, w in enumerate(e.layers):
            kc, vc = self.cache[i, 0], self.cache[i, 1]
            e._norm_fwd(h, w.g1, w.b1, ln, m, r)
            self._linear(ln, w.wqkv, w.bqkv, qkv)
            self._qkv_post(w, qkv, x.get("qk_pre"), x.get("qk_tmp"), m, r)
            ops.decode_append(qkv, pos, kc, vc, e.rope, c.n_heads, slot, n_kv_heads=c.kv_n_heads)
            if tiles is None:
                ops.decode_attention(qkv, kc, vc, pos, attn, c.n_heads, self.scale, e.alibi, n_kv_heads=c.kv_n_heads,
                                     window=self.window)
            else:
                ops.cache_attention(qkv, kc, vc, tiles, attn, c.n_heads, self.scale, e.alibi, n_kv_heads=c.kv_n_heads,
                                    window=self.window)
            self._linear(attn, w.wo, w.bo, hmid, residual=h)
            e._norm_fwd(hmid, w.g2, w.b2, ln, m, r)
            self._ffn(w, ln, u, z, h, hmid, x.get("ffn_d"), x.get("ffn_c"))

    # --------------------------------------------------------------------- step
    def _step_kernels(self, b: int) -> None:
        e, B = self.e, self.buf
        x = {k: v[:b] for k, v in B.items() if k != "logits"}
        ops.embed_pos(self.tok, self.pos, e.wte16, e.wpe16, x["h"])
        self._blocks(x, self.pos)
        e._norm_fwd(x["h"], e.gf, e.bf, x["ln"], x["m"], x["r"])
        self._linear(x["ln"], e.head16, None, B["logits"][:b])
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

    # ------------------------------------------------------------------ scoring
    @torch.no_grad()
    def score(self, pairs: list[tuple[list[int], list[int]]]) -> list[tuple[float, bool]]:
        """Log-likelihood of each pair's scored tokens after its context: ``[(sum log p(scored | context), every scored token is
        the argmax)]``. Pairs that share a context share one prefill; each pair holds one cache slot, so a call takes at most
        ``max_batch`` pairs. Contexts and scored tokens are taken as given (no truncation). Eager: shapes change every call.

        Steps: (1) prefill every distinct context once, into the slot of its first pair; (2) the last context row's logits
        score ``scored[0]`` of every pair of the group; (3) the context k / v is copied into the slot of every other pair of
        the group; (4) ``scored[:-1]`` of every pair run through the blocks at positions ``P ..`` of its slot (cache attention);
        (5) final LN + LM head over all those rows, log p and the argmax match of each scored token on the device, one copy to
        the host, and each pair's tokens summed in order there."""
        c, e = self.cfg, self.e
        if not 1 <= len(pairs) <= self.max_batch:
            raise ValueError(f"{len(pairs)} pairs; this decoder scores 1..{self.max_batch} at a time")
        for ctx, sc in pairs:
            if not ctx or not sc:
                raise ValueError("every scored pair needs a non-empty context and at least one scored token")
            if len(ctx) + len(sc) > self.max_seq_len:
                raise ValueError(f"a context of {len(ctx)} plus {len(sc)} scored tokens does not fit the {self.max_seq_len}-position cache")
        self._ensure_capacity(len(pairs))
        self._b = 0   # the slots are overwritten: a generation started before cannot step on
        groups: dict[tuple[int, ...], list[int]] = {}
        for i, (ctx, _) in enumerate(pairs):
            groups.setdefault(tuple(ctx), []).append(i)
        members = list(groups.values())
        G = len(members)
        last = self._prefill([pairs[g[0]][0] for g in members], [g[0] for g in members])
        for g in members:
            P = len(pairs[g[0]][0])
            for i in g[1:]:
                self.cache[:, :, i, :, :P].copy_(self.cache[:, :, g[0], :, :P])
        # extend rows: scored[:-1] of every pair at positions P .. P + n - 2 of its slot (the last scored token is no input)
        toks: list[int] = []
        pos: list[int] = []
        runs: list[tuple[int, int, int, int]] = []
        first = [0] * len(pairs)
        for i, (ctx, sc) in enumerate(pairs):
            first[i] = G + len(toks)
            if len(sc) > 1:
                runs.append((i, len(toks), len(sc) - 1, len(ctx)))
                toks += sc[:-1]
                pos += range(len(ctx), len(ctx) + len(sc) - 1)
        R = G + len(toks)
        hid = torch.empty(R, c.d_model, dtype=torch.bfloat16, device=self.dev)
        hid[:G].copy_(last)
        if toks:
            x = self._row_buffers(len(toks), h=hid[G:])
            i32 = lambda v: torch.tensor(v, dtype=torch.int32).to(self.dev, non_blocking=True)  # noqa: E731
            pos_t = i32(pos)
            ops.embed_pos(i32(toks), pos_t, e.wte16, e.wpe16, x["h"])
            self._blocks(x, pos_t, i32([s for s, _, n, _ in runs for _ in range(n)]), ops.cache_tiles(runs, self.dev))
        ln = torch.empty_like(hid)
        m, r = (torch.empty(R, dtype=torch.float32, device=self.dev) for _ in range(2))
        e._norm_fwd(hid, e.gf, e.bf, ln, m, r)
        logits = torch.empty(R, c.vocab_size, dtype=torch.bfloat16, device=self.dev)
        self._linear(ln, e.head16, None, logits)
        # scored token k of pair i is predicted by its group's last context row (k = 0) or by extend row first[i] + k - 1
        group = {i: gi for gi, g in enumerate(members) for i in g}
        rows = [group[i] if k == 0 else first[i] + k - 1 for i, (_, sc) in enumerate(pairs) for k in range(len(sc))]
        tgts = [t for _, sc in pairs for t in sc]
        lse = torch.empty(R, dtype=torch.float32, device=self.dev)
        stats = torch.zeros(4, dtype=torch.float64, device=self.dev)
        # log p = T(logit) - lse(T(logits)) with the head's transform T (logit_scale / final_logit_softcapping); the argmax of
        # the raw logits is that of T(logits): T is strictly increasing
        ops.cross_entropy(logits, torch.full((R,), -1, dtype=torch.long, device=self.dev), 0.0, False, stats, row_lse=lse,
                          logit_scale=e.head_scale, softcap=e.head_cap)
        top = torch.empty(R, dtype=torch.int32, device=self.dev)
        ops.argmax_advance(logits, top)
        row_t = torch.tensor(rows, dtype=torch.long).to(self.dev, non_blocking=True)
        tgt_t = torch.tensor(tgts, dtype=torch.long).to(self.dev, non_blocking=True)
        logp = head_transform(logits[row_t, tgt_t].float(), e.head_scale, e.head_cap) - lse[row_t]
        host = torch.stack([logp, (top[row_t].long() == tgt_t).float()]).cpu().tolist()
        out, k = [], 0
        for _, sc in pairs:
            total, hit = 0.0, True
            for _ in sc:
                total += host[0][k]
                hit = hit and host[1][k] == 1.0
                k += 1
            out.append((total, hit))
        return out

    def close(self) -> None:
        self._graphs.clear()
        self.cache = None
        self.buf = {}
        self._cap = self._b = 0
