"""Reference attention for the kernel tests: an fp64 oracle, a bf16 baseline, and a per-tile acceptance criterion.

* ``oracle``: explicit attention in float64 on the bf16 inputs (upcast), one (batch, head) at a time so the S x S matrices
  stay small. Returns O, the natural-log LSE and, given dO, dQ / dK / dV from fp64 autograd.
* ``baseline``: the same explicit math run in bf16 by PyTorch (``q @ k^T * scale``, bias, mask, softmax, ``@ v``, autograd).
  Its distance from the oracle is the error bf16 arithmetic makes at that exact input.
* ``check``: each tile of a kernel result must satisfy
  ``max|kernel - oracle| <= 2 * max|baseline - oracle| + 1e-5 * max|oracle|`` and
  ``mean|kernel - oracle| <= 1.25 * mean|baseline - oracle| + 1e-5 * max|oracle|``, both over the tile, and over the whole
  tensor ``mean|kernel - oracle| <= mean|baseline - oracle|``. The kernels keep scores and the softmax in fp32, so they must
  be at least as accurate as bf16 math on average. The tile-max part alone lets a 2 % scaling of one dQ tile through (its
  error sits at about 1.0x its bound) and so does the whole-tensor mean; the tile mean sees it 3-6x over the baseline's
  with N(0, 1) inputs.
* ``KNOWN``: input cases where the H100 kernels measurably miss the bound, with the cause. ``check`` reports those as an
  expected failure (after every other check of the test has run) instead of widening the bound for everyone.

Tensors are per head: ``[B, H, R, dh]``. Rows are query positions for O and dQ, key positions for dK and dV.
"""
from __future__ import annotations

import math
from dataclasses import dataclass

import torch

TILE = 128          # rows per tile of the training kernels (query tiles forward, key tiles backward)
TILE_SLACK = 2.0    # kernel tile error may be this many times the bf16 baseline's
FLOOR = 1e-5        # ... plus this fraction of the tile's largest |oracle| (exact-zero and exactly representable tiles)
# mean error per tile may be this many times the baseline's; over the whole tensor it may not exceed it. Measured on an H100
# (700 W): with ALiBi and q = 0 the forward's worst tile mean is 1.11x the baseline's, its whole-tensor mean 0.83x
TILE_MEAN_SLACK = 1.25
CASES = ("normal", "peaked", "rising", "uniform")


# ------------------------------------------------------------------------------------------------ inputs
def make_inputs(case: str, B: int, S: int, H: int, dh: int, device, seed: int = 0) -> tuple[torch.Tensor, torch.Tensor]:
    """bf16 ``qkv`` [B, S, 3*H*dh] and ``dout`` [B, S, H*dh] for one input case.

    normal : N(0, 1).
    peaked : q and k x3, so each softmax row is close to one-hot.
    rising : q and k share a direction u and k grows along it with the key index; the score rises by about 0.5 per
             128-key tile (plus small noise), so every new KV tile raises the running max and the online rescale runs
             on every tile.
    uniform: q = 0, so every score is 0 and O is a running mean of V.
    """
    g = torch.Generator(device="cpu").manual_seed(seed)
    d = H * dh
    x = torch.randn(B, S, 3, H, dh, generator=g)
    dout = torch.randn(B, S, d, generator=g)
    if case == "peaked":
        x[:, :, :2] *= 3.0
    elif case == "rising":
        u = torch.ones(dh) / math.sqrt(dh)
        per_tile = 0.5 * math.sqrt(dh)   # q.k rise per 128 keys before the 1/sqrt(dh) scale
        a = 2.0
        ramp = torch.arange(S, dtype=torch.float32) / TILE * (per_tile / a)
        x[:, :, 0] = 0.1 * x[:, :, 0] + a * u
        x[:, :, 1] = 0.1 * x[:, :, 1] + ramp[None, :, None, None] * u
    elif case == "uniform":
        x[:, :, 0] = 0.0
    elif case != "normal":
        raise ValueError(case)
    return x.reshape(B, S, 3 * d).to(device).bfloat16(), dout.to(device).bfloat16()


def split_heads(qkv: torch.Tensor, H: int) -> tuple[torch.Tensor, torch.Tensor, torch.Tensor]:
    """[B, S, 3*H*dh] -> q, k, v each [B, H, S, dh] (views)."""
    B, S, D3 = qkv.shape
    q, k, v = qkv.view(B, S, 3, H, D3 // (3 * H)).permute(2, 0, 3, 1, 4)
    return q, k, v


def heads(x: torch.Tensor, H: int) -> torch.Tensor:
    """[B, S, H*dh] -> [B, H, S, dh] (view)."""
    B, S, d = x.shape
    return x.view(B, S, H, d // H).transpose(1, 2)


# ------------------------------------------------------------------------------------------------ attention math
def _bias_mask(q_pos: torch.Tensor, k_pos: torch.Tensor, causal: bool, slope: float | None, dtype) -> tuple[torch.Tensor | None, torch.Tensor | None]:
    rel = (k_pos[None, :] - q_pos[:, None]).to(dtype)
    bias = slope * rel if slope is not None else None
    keep = (k_pos[None, :] <= q_pos[:, None]) if causal else None
    return bias, keep


def attend(q, k, v, scale: float, *, causal: bool, slope: float | None = None, q_pos=None, keep=None, dout=None):
    """Explicit attention of one head in the dtype of its inputs: q [R, dh] at positions ``q_pos`` (default 0..R-1),
    k / v [N, dh] at positions 0..N-1. ``keep`` [R, N] overrides the causal mask. Returns (O, LSE, (dq, dk, dv) or None)."""
    R, N = q.shape[0], k.shape[0]
    q_pos = torch.arange(R, device=q.device) if q_pos is None else q_pos
    k_pos = torch.arange(N, device=q.device)
    bias, causal_keep = _bias_mask(q_pos, k_pos, causal, slope, q.dtype)
    keep = causal_keep if keep is None else keep
    with torch.enable_grad():
        leaves = [t.detach().requires_grad_(dout is not None) for t in (q, k, v)]
        s = (leaves[0] @ leaves[1].t()) * scale
        if bias is not None:
            s = s + bias
        if keep is not None:
            s = s.masked_fill(~keep, float("-inf"))
        lse = torch.logsumexp(s.detach().double(), -1)
        o = torch.softmax(s, -1) @ leaves[2]
        grads = torch.autograd.grad(o, leaves, dout) if dout is not None else None
    return o.detach(), lse, grads


@dataclass
class Result:
    o: torch.Tensor                       # [B, H, R, dh]
    lse: torch.Tensor | None = None       # [B, H, R] (oracle only)
    dq: torch.Tensor | None = None        # [B, H, R, dh]
    dk: torch.Tensor | None = None        # [B, H, N, dh]
    dv: torch.Tensor | None = None


def _run(q, k, v, dout, scale, causal, slopes, q_pos, lengths, dtype, keep_fn=None) -> Result:
    """Loop over (batch, head). q [B, H, R, dh]; k, v [B, H, N, dh]; q_pos [B, R] or None; lengths[b]: keys of batch row b
    (default all N); slopes: per-head floats or None; keep_fn(b, h, q_pos, n) -> [R, n] mask override (perturbed oracles)."""
    B, H, R, dh = q.shape
    N = k.shape[2]
    o = torch.zeros(B, H, R, dh, dtype=torch.float64, device=q.device)
    lse = torch.zeros(B, H, R, dtype=torch.float64, device=q.device)
    grads = None if dout is None else [torch.zeros(B, H, n, dh, dtype=torch.float64, device=q.device) for n in (R, N, N)]
    for b in range(B):
        n = N if lengths is None else int(lengths[b])
        qp = None if q_pos is None else q_pos[b]
        for h in range(H):
            keep = None if keep_fn is None else keep_fn(b, h, qp if qp is not None else torch.arange(R, device=q.device), n)
            res = attend(q[b, h].to(dtype), k[b, h, :n].to(dtype), v[b, h, :n].to(dtype), scale, causal=causal,
                         slope=None if slopes is None else float(slopes[h]), q_pos=qp, keep=keep,
                         dout=None if dout is None else dout[b, h].to(dtype))
            o[b, h] = res[0].double()
            lse[b, h] = res[1]
            if grads is not None:
                for dst, gsrc in zip(grads, res[2]):
                    dst[b, h, : gsrc.shape[0]] = gsrc.double()
    r = Result(o, lse)
    if grads is not None:
        r.dq, r.dk, r.dv = grads
    return r


def oracle(q, k, v, scale: float, *, causal: bool, slopes=None, dout=None, q_pos=None, lengths=None, keep_fn=None) -> Result:
    """fp64 attention of bf16 (or any) inputs, per head. See ``_run`` for the layouts."""
    return _run(q, k, v, dout, scale, causal, slopes, q_pos, lengths, torch.float64, keep_fn)


def baseline(q, k, v, scale: float, *, causal: bool, slopes=None, dout=None, q_pos=None, lengths=None) -> Result:
    """The same explicit math in bf16 (PyTorch ops, bf16 outputs at every step). Its lse is not used."""
    if q_pos is None and lengths is None:
        return _baseline_batched(q, k, v, scale, causal, slopes, dout)
    return _run(q, k, v, dout, scale, causal, slopes, q_pos, lengths, torch.bfloat16)


def _baseline_batched(q, k, v, scale, causal, slopes, dout) -> Result:
    """All heads at once (bf16 S x S scores are a quarter of the fp64 ones); same ops as ``attend``."""
    B, H, S, dh = q.shape
    pos = torch.arange(S, device=q.device)
    with torch.enable_grad():
        leaves = [t.detach().bfloat16().requires_grad_(dout is not None) for t in (q, k, v)]
        s = (leaves[0] @ leaves[1].transpose(-1, -2)) * scale
        if slopes is not None:
            rel = (pos[None, :] - pos[:, None]).bfloat16()
            s = s + torch.as_tensor(slopes, dtype=torch.float32).to(q.device).bfloat16()[:, None, None] * rel
        if causal:
            s = s.masked_fill(pos[None, :] > pos[:, None], float("-inf"))
        o = torch.softmax(s, -1) @ leaves[2]
        grads = torch.autograd.grad(o, leaves, dout.bfloat16()) if dout is not None else None
    r = Result(o.detach().double())
    if grads is not None:
        r.dq, r.dk, r.dv = (t.double() for t in grads)
    return r


# ------------------------------------------------------------------------------------------------ criterion
def tile_report(name: str, got: torch.Tensor, ref: torch.Tensor, base: torch.Tensor, rows: int = TILE, case: str = "",
                whole_mean: bool = False) -> dict:
    """Evaluate the criterion without asserting. got / ref / base: [B, H, R, dh] (any float dtype); tiles of ``rows`` rows
    (R % rows == 0). Returns the worst tile's ratio to its max bound, the worst mean ratio and a message naming the tiles.
    ``whole_mean``: take the mean part over the whole tensor instead of per tile (single-row tiles of decode attention,
    where 64 or 128 rounding errors are too few for a per-row mean to be stable; cache-attention tiles of unequal size)."""
    got, ref, base = got.double(), ref.double(), base.double()
    B, H, R, dh = ref.shape
    assert got.shape == ref.shape == base.shape, (name, got.shape, ref.shape, base.shape)
    assert R % rows == 0, (name, R, rows)
    ek = (got - ref).abs().reshape(B, H, R // rows, rows * dh)
    eb = (base - ref).abs().reshape(B, H, R // rows, rows * dh)
    mag = ref.abs().reshape(B, H, R // rows, rows * dh).amax(-1)

    def ratio(err, bound):
        return torch.where(bound > 0, err / bound, torch.where(err > 0, torch.full_like(err, math.inf), torch.zeros_like(err)))

    k_max, b_max = ek.amax(-1), eb.amax(-1)
    bound = TILE_SLACK * b_max + FLOOR * mag
    over = ratio(k_max, bound)
    if whole_mean:
        k_mean, b_mean, mag_all = ek.mean().reshape(1, 1, 1), eb.mean().reshape(1, 1, 1), mag.amax().reshape(1, 1, 1)
        mean_bound = b_mean + FLOOR * mag_all
    else:
        k_mean, b_mean = ek.mean(-1), eb.mean(-1)
        mean_bound = TILE_MEAN_SLACK * b_mean + FLOOR * mag
    mean_over = ratio(k_mean, mean_bound)
    whole_k, whole_b = ek.mean().item(), eb.mean().item()
    whole_ratio = whole_k / (whole_b + FLOOR * mag.amax().item()) if whole_k > 0 else 0.0
    nan = bool(torch.isnan(got).any())

    def where(r):
        return tuple(int(i) for i in torch.unravel_index(r.argmax(), r.shape))

    b, h, t = where(over)
    mb, mh, mt = where(mean_over)
    msg = (f"{name} [{case}]: worst tile (b={b}, h={h}, tile={t}) max err {k_max[b, h, t].item():.3e} vs bound "
           f"{bound[b, h, t].item():.3e} (baseline {b_max[b, h, t].item():.3e}, ratio {over[b, h, t].item():.2f}); "
           f"worst tile mean (b={mb}, h={mh}, tile={mt}) err {k_mean[mb, mh, mt].item():.3e} vs bound {mean_bound[mb, mh, mt].item():.3e} "
           f"(ratio {mean_over[mb, mh, mt].item():.2f}); whole-tensor mean err {whole_k:.3e} vs baseline {whole_b:.3e} "
           f"(ratio {whole_ratio:.2f})"
           + ("; NaN in kernel output" if nan else ""))
    worst_mean = max(mean_over[mb, mh, mt].item(), whole_ratio)
    return {"tile_ratio": math.inf if nan else over[b, h, t].item(), "mean_ratio": math.inf if nan else worst_mean, "msg": msg}


# (tensor, input case) -> why the H100 kernel misses the bound there. Measured on an H100 80GB HBM3 at 700 W.
KNOWN = {
    ("dq", "rising"): "training backward dQ on rising scores with ALiBi: worst tile max 1.26x its bound, worst tile mean 2.3x "
                      "and whole-tensor mean 1.54x the baseline's. delta = rowsum(dO * O) is taken from the bf16-rounded O, so "
                      "the rows of dS do not sum to zero and the residual multiplies the keys' common component, which the "
                      "rising input makes large (|k| up to ~45). The kernel's dQ equals an fp32 emulation of its own math; in "
                      "that emulation, delta from the exact O instead of the bf16 O lowers the whole-tensor mean ratio from "
                      "0.92 to 0.62 (d_head 64, causal, S = 2048)",
}


class Deviations(list):
    """Known misses collected by ``check`` during a test; ``report()`` at its end turns them into an expected failure."""

    def report(self):
        if self:
            import pytest

            pytest.xfail("known deviation from the bf16 bound: " + " | ".join(self))


def check(name: str, got, ref, base, rows: int = TILE, case: str = "", whole_mean: bool = False,
          deviations: Deviations | None = None) -> dict:
    """Assert the per-tile max and mean criterion (see the module docstring). A miss listed in ``KNOWN`` for (name, input
    case) goes to ``deviations`` instead, if given; NaN never does."""
    rep = tile_report(name, got, ref, base, rows, case, whole_mean)
    print(rep["msg"])
    ok = rep["tile_ratio"] <= 1.0 and rep["mean_ratio"] <= 1.0
    known = KNOWN.get((name, case.split(",")[0]))
    if not ok and known and deviations is not None and math.isfinite(rep["tile_ratio"]) and math.isfinite(rep["mean_ratio"]):
        deviations.append(f"{known}: {rep['msg']}")
        return rep
    assert rep["tile_ratio"] <= 1.0 and rep["mean_ratio"] <= 1.0, rep["msg"]
    return rep


def check_tiles(name: str, got: list, ref: list, base: list, case: str = "") -> None:
    """Tiles of different sizes (the cache-attention tile table): each list entry is one tile ``[1, H, n, dh]``. The max part
    is applied per (tile, head), the mean part over all tiles together."""
    for i, (g, r, b) in enumerate(zip(got, ref, base)):
        rep = tile_report(name, g, r, b, rows=r.shape[2], case=f"{case}, tile {i}", whole_mean=True)
        assert rep["tile_ratio"] <= 1.0, rep["msg"]
    rep = tile_report(name, torch.cat(got, 2), torch.cat(ref, 2), torch.cat(base, 2), rows=1, case=case, whole_mean=True)
    print(rep["msg"])
    assert rep["mean_ratio"] <= 1.0, rep["msg"]


def check_lse(got: torch.Tensor, ref: torch.Tensor, atol: float, case: str = "") -> float:
    """fp32 LSE (never rounded to bf16) element by element against the fp64 oracle. Returns the max error."""
    err = (got.double() - ref.double()).abs()
    worst = int(err.argmax()) if err.numel() else 0
    e = err.flatten()[worst].item() if err.numel() else 0.0
    print(f"lse [{case}]: max err {e:.3e} (bound {atol:.1e})")
    assert not torch.isnan(got).any() and e <= atol, (
        f"lse [{case}]: element {tuple(int(i) for i in torch.unravel_index(torch.tensor(worst), err.shape))} err {e:.3e} > {atol:.1e}")
    return e
