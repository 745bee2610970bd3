"""The attention acceptance criterion on CPU: it accepts a healthy kernel stand-in and rejects small confined errors.

The stand-in is fp32 attention math with its outputs rounded to bf16 (what a healthy fp32-softmax kernel computes, minus
the bf16 P operand). Each perturbation is a copy of the fp64 oracle's output with one of the errors an attention kernel
can make in a single tile or on a mask edge; the criterion must reject every one of them.
"""
import functools
import math

import pytest
import torch

import attention_oracle as A

H = 2   # head 1 carries the smallest ALiBi slope of a 12-head model


def _slopes():
    from photon_b200.models.mpt import alibi_slopes

    return alibi_slopes(12)[[0, -1]].tolist()


@functools.lru_cache(maxsize=None)
def _setup(S, dh, alibi):
    qkv, dout = A.make_inputs("normal", 1, S, H, dh, "cpu", seed=S + dh)
    q, k, v = A.split_heads(qkv, H)
    do = A.heads(dout, H)
    slopes = _slopes() if alibi else None
    scale = 1.0 / math.sqrt(dh)
    kw = dict(causal=True, slopes=slopes, dout=do)
    ref = A.oracle(q, k, v, scale, **kw)
    base = A.baseline(q, k, v, scale, **kw)
    return (q, k, v, do, scale, slopes), ref, base


def _failures(got: A.Result, ref: A.Result, base: A.Result) -> list[str]:
    out = []
    for n in ("o", "dq", "dk", "dv"):
        rep = A.tile_report(n, getattr(got, n), getattr(ref, n), getattr(base, n))
        if rep["tile_ratio"] > 1.0 or rep["mean_ratio"] > 1.0:
            out.append(rep["msg"])
    return out


SHAPES = [(384, 64), (384, 128), (2048, 64), (2048, 128)]


@pytest.mark.parametrize("alibi", [False, True])
@pytest.mark.parametrize("S,dh", SHAPES)
def test_fp32_standin_is_accepted(S, dh, alibi):
    (q, k, v, do, scale, slopes), ref, base = _setup(S, dh, alibi)
    st = A._run(q, k, v, do, scale, True, slopes, None, None, torch.float32)
    rounded = A.Result(*(t.bfloat16().double() for t in (st.o, st.lse, st.dq, st.dk, st.dv)))
    for n in ("o", "dq", "dk", "dv"):
        A.check(n, getattr(rounded, n), getattr(ref, n), getattr(base, n), case=f"fp32 stand-in S={S} dh={dh}")


def _perturbed(kind, S, dh):
    alibi = kind == "alibi_slope"
    (q, k, v, do, scale, slopes), ref, base = _setup(S, dh, alibi)
    pos = torch.arange(S)
    if kind == "dkdv_last_tile_zero":
        dk, dv = ref.dk.clone(), ref.dv.clone()
        dk[:, :, -A.TILE:] = 0
        dv[:, :, -A.TILE:] = 0
        return A.Result(ref.o, ref.lse, ref.dq, dk, dv), ref, base
    if kind == "dq_tile_x1.02":
        dq = ref.dq.clone()
        dq[:, :, -A.TILE:] *= 1.02
        return A.Result(ref.o, ref.lse, dq, ref.dk, ref.dv), ref, base
    if kind == "key_hidden_from_later_tiles":
        hidden = torch.zeros(S, S, dtype=torch.bool)
        for t in range(S // A.TILE):
            hidden[(t + 1) * A.TILE:, t * A.TILE + 37] = True   # key 37 of tile t, for every query of a later tile

        def keep_fn(b, h, qp, n):
            return (pos[None, :] <= pos[:, None]) & ~hidden
    elif kind == "causal_diagonal_dropped":
        def keep_fn(b, h, qp, n):
            keep = pos[None, :] < pos[:, None]
            keep[0, 0] = True   # row 0 keeps its only key, so no row is empty
            return keep
    elif kind == "alibi_slope":
        slopes = list(slopes)
        slopes[-1] *= 1.05
        keep_fn = None
    else:
        raise ValueError(kind)
    got = A.oracle(q, k, v, scale, causal=True, slopes=slopes, dout=do, keep_fn=keep_fn)
    return got, ref, base


@pytest.mark.parametrize("kind", ["dkdv_last_tile_zero", "key_hidden_from_later_tiles", "dq_tile_x1.02", "causal_diagonal_dropped",
                                  "alibi_slope"])
@pytest.mark.parametrize("S,dh", SHAPES)
def test_perturbation_is_rejected(S, dh, kind):
    got, ref, base = _perturbed(kind, S, dh)
    assert _failures(got, ref, base), f"{kind} at S={S} dh={dh} passed the criterion"


def test_failure_message_names_the_tile():
    (q, k, v, do, scale, slopes), ref, base = _setup(384, 64, False)
    dk = ref.dk.clone()
    dk[0, 1, 2 * A.TILE + 5] += 1.0
    with pytest.raises(AssertionError, match=r"dk \[probe\]: worst tile \(b=0, h=1, tile=2\)"):
        A.check("dk", dk, ref.dk, base.dk, case="probe")


def test_lse_check_is_elementwise():
    ref = torch.zeros(1, 2, 256, dtype=torch.float64)
    got = ref.clone().float()
    A.check_lse(got, ref, 1e-5)
    got[0, 1, 200] = 2e-5
    with pytest.raises(AssertionError, match=r"element \(0, 1, 200\)"):
        A.check_lse(got, ref, 1e-5)
