"""The GEMM epilogues write through shared memory and TMA stores: every accepted (A layout, B layout, epilogue, operand type)
combination with cluster 1 and 2, on tails in M, N and K, into a column slice of a wider buffer. Checked against an fp32
reference, for untouched guard rows / columns around the output, and for bitwise-equal repeated runs."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

EPI_BF16, EPI_RESIDUAL, EPI_GELU_DUAL, EPI_DGELU, EPI_F32, EPI_GELU_GRAD, EPI_MUL, EPI_GELU_GRAD_Q8 = range(8)
CASES = [(0, 0, EPI_BF16, 0), (0, 0, EPI_RESIDUAL, 0), (0, 0, EPI_GELU_DUAL, 0), (0, 0, EPI_F32, 0), (0, 1, EPI_BF16, 0),
         (0, 1, EPI_DGELU, 0), (0, 1, EPI_MUL, 0), (0, 0, EPI_GELU_GRAD, 0), (0, 1, EPI_F32, 0), (1, 1, EPI_F32, 0),
         (1, 1, EPI_BF16, 0), (1, 0, EPI_F32, 0), (1, 0, EPI_BF16, 0),
         (0, 0, EPI_BF16, 1), (0, 0, EPI_RESIDUAL, 1), (0, 0, EPI_GELU_GRAD, 1), (0, 0, EPI_GELU_GRAD_Q8, 1), (0, 0, EPI_F32, 1),
         (0, 0, EPI_MUL, 1)]
# M: an odd number of M tiles with a tail / a single partial tile; N % 256 != 0 and N % 64 != 0; K tails for both k-block widths
SHAPES = [(520, 328, 208), (72, 584, 144)]
OFF = 32                   # output = columns [OFF, OFF + N) of rows [0, M) in an [M + 8, N + pad] buffer, rows of 16-byte pieces
Q8_SCALE = 16.0


def _dev():
    return torch.device("cuda", 0)


def _gelu_grad(z):
    return 0.5 * (1 + torch.erf(z / math.sqrt(2))) + z * torch.exp(-0.5 * z * z) / math.sqrt(2 * math.pi)


def _run(amn, bmn, epi, fp8, M, N, K, cluster):
    from photon_b200 import ops

    gen = torch.Generator(device=_dev())
    gen.manual_seed(7)
    dev = _dev()
    a = (torch.randn(*((K, M) if amn else (M, K)), device=dev, generator=gen)).to(torch.bfloat16)
    b = (torch.randn(*((K, N) if bmn else (N, K)), device=dev, generator=gen) * 0.05).to(torch.bfloat16)
    a_fmt = ops.E5M2 if (amn or bmn) else ops.E4M3
    if fp8:
        a8 = a.float().to(torch.float8_e5m2 if a_fmt == ops.E5M2 else torch.float8_e4m3fn)
        b8 = b.float().to(torch.float8_e4m3fn)
        af, bf = a8.float(), b8.float()
        a, b = a8.view(torch.uint8), b8.view(torch.uint8)
    else:
        af, bf = a.float(), b.float()
    acc = (af.t() if amn else af) @ (bf if bmn else bf.t())
    f32 = epi == EPI_F32
    bias = None if f32 else torch.randn(N, device=dev, generator=gen) * 0.1
    aux = torch.randn(M, N, device=dev, generator=gen).to(torch.bfloat16) if epi in (EPI_RESIDUAL, EPI_DGELU, EPI_MUL) else None
    z = acc + (bias if bias is not None else 0)
    pad = 64 - N % 16

    def buf(dtype):
        if dtype == torch.uint8:
            return torch.full((M + 8, N + pad), 0x7E, device=dev, dtype=torch.uint8)
        return torch.full((M + 8, N + pad), -7.0, device=dev, dtype=dtype)

    outs = {"D": buf(torch.float32 if f32 else torch.bfloat16)}
    if f32:
        outs["D"].zero_()
    if epi in (EPI_GELU_DUAL, EPI_GELU_GRAD, EPI_GELU_GRAD_Q8):
        outs["D2"] = buf(torch.bfloat16)
    if epi == EPI_GELU_GRAD_Q8:
        outs["D8"] = buf(torch.uint8)
    guards = {k: v.clone() for k, v in outs.items()}
    view = {k: v[:M, OFF:OFF + N] for k, v in outs.items()}
    kw = dict(a_mn=bool(amn), b_mn=bool(bmn), epi=epi, bias=bias, aux=aux, out2=view.get("D2"), accumulate=f32, cluster=cluster)
    meta = None
    if fp8:
        meta = torch.ones(3, 3, device=dev)
        meta[0, 2], meta[1, 2], meta[2, 2] = Q8_SCALE, 1 / Q8_SCALE, 0.0
        d = view["D2"] if epi == EPI_GELU_GRAD_Q8 else view["D"]
        ops.gemm_fp8(a, b, d, meta, 0, 1, a_fmt=a_fmt, b_fmt=ops.E4M3, out8=view.get("D8"), role_out=2, **kw)
    else:
        ops.gemm(a, b, view["D"], **kw)
    torch.cuda.synchronize()
    refs = {}
    if f32:
        refs["D"] = acc
    elif epi == EPI_BF16:
        refs["D"] = z
    elif epi == EPI_RESIDUAL:
        refs["D"] = z + aux.float()
    elif epi == EPI_MUL:
        refs["D"] = z * aux.float()
    elif epi == EPI_DGELU:
        refs["D"] = z * _gelu_grad(aux.float())
    elif epi == EPI_GELU_DUAL:
        refs["D"], refs["D2"] = torch.nn.functional.gelu(z), z
    else:
        refs["D2"] = _gelu_grad(z)
        if epi == EPI_GELU_GRAD:
            refs["D"] = torch.nn.functional.gelu(z)
        else:
            refs["D8"] = torch.nn.functional.gelu(z)
    return outs, guards, view, refs, meta


@pytest.mark.parametrize("M,N,K", SHAPES)
@pytest.mark.parametrize("cluster", [1, 2])
@pytest.mark.parametrize("amn,bmn,epi,fp8", CASES)
def test_gemm_epilogue(amn, bmn, epi, fp8, cluster, M, N, K):
    if epi == EPI_GELU_GRAD_Q8:
        N += 8             # E4M3 rows must be whole 16-byte pieces; still N % 64 != 0
    outs, guards, view, refs, meta = _run(amn, bmn, epi, fp8, M, N, K, cluster)
    for k, buf in outs.items():
        # everything outside the [M, N] window is untouched
        inside = torch.zeros(buf.shape, dtype=torch.bool, device=buf.device)
        inside[:M, OFF:OFF + N] = True
        assert torch.equal(buf[~inside], guards[k][~inside]), f"{k}: the epilogue wrote outside its output"
    for k, ref in refs.items():
        if k == "D8":
            got = view[k].view(torch.float8_e4m3fn).float() / Q8_SCALE
            rtol, atol = 0.07, 2e-3
        else:
            got = view[k].float()
            rtol, atol = (1e-2, 5e-2) if epi == EPI_F32 else (2e-2, 3e-2)
        err = (got - ref).abs()
        bad = int((err > atol + rtol * ref.abs()).sum())
        assert bad == 0, f"{k}: {bad} of {err.numel()} elements out of tolerance, max err {err.max().item():.4g}"
    if meta is not None and epi == EPI_GELU_GRAD_Q8:
        want = refs["D8"].abs().max().item()
        assert abs(meta[2, 2].item() - want) <= 1e-2 * want, (meta[2, 2].item(), want)
    # a second run writes the same bits
    outs2, _, _, _, _ = _run(amn, bmn, epi, fp8, M, N, K, cluster)
    for k in outs:
        assert torch.equal(outs[k], outs2[k]), f"{k}: two runs differ"


@pytest.mark.parametrize("N,pad", [(256, 8), (264, 8)])
def test_gemm_fp8_output_needs_16_byte_rows(N, pad):
    """The E4M3 output is stored by TMA in 16-byte pieces: its row stride and N must be multiples of 16 bytes."""
    from photon_b200 import ops

    dev = _dev()
    M, K = 128, 128
    a = torch.zeros(M, K, device=dev, dtype=torch.uint8)
    b = torch.zeros(N, K, device=dev, dtype=torch.uint8)
    d2 = torch.empty(M, N, device=dev, dtype=torch.bfloat16)
    d8 = torch.empty(M, N + pad, device=dev, dtype=torch.uint8)[:, :N]
    meta = torch.ones(3, 3, device=dev)
    with pytest.raises(RuntimeError, match="16"):
        ops.gemm_fp8(a, b, d2, meta, 0, 1, epi=ops.EPI_GELU_GRAD_Q8, out2=d2, out8=d8, role_out=2)
