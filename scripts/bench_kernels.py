"""Kernel microbenchmarks on one GPU: our wgmma GEMM vs cuBLAS (torch.matmul) on the MPT shapes,
bandwidth of the fused memory-bound kernels. CUDA-event timed, L2 flushed between iterations."""
import json
import sys
import time
from pathlib import Path

import torch

sys.path.insert(0, str(Path(__file__).resolve().parents[1]))
from photon_b200 import ops  # noqa: E402
from photon_b200.utils.hw import measured_peaks  # noqa: E402

dev = torch.device("cuda", 0)
flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)


def timeit(fn, iters=10, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(iters):
        flush.zero_()
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        fn()
        e.record()
        torch.cuda.synchronize()
        ts.append(s.elapsed_time(e))
    ts.sort()
    return ts[len(ts) // 2]


def main():
    pk = measured_peaks()
    rows = []
    T = 32768
    d1 = 2048   # MPT-1B geometry (BASELINE config #4)
    shapes = [("1b qkv fwd", 16384, 3 * d1, d1, 0, 0), ("1b up fwd", 16384, 4 * d1, d1, 0, 0), ("1b down fwd", 16384, d1, 4 * d1, 0, 0),
              ("1b up dgrad", 16384, d1, 4 * d1, 0, 1), ("1b up wgrad", 4 * d1, d1, 16384, 1, 1),
              ("qkv fwd", T, 2304, 768, 0, 0), ("out fwd", T, 768, 768, 0, 0), ("up fwd", T, 3072, 768, 0, 0),
              ("down fwd", T, 768, 3072, 0, 0), ("up dgrad", T, 768, 3072, 0, 1), ("up wgrad", 3072, 768, T, 1, 1),
              ("lmhead fwd", 8192, 50368, 768, 0, 0), ("lmhead dgrad", 8192, 768, 50368, 0, 1), ("lmhead wgrad", 50368, 768, 8192, 1, 1),
              # the shapes the engine ACTUALLY issues for the head: chunks of 16896 rows = 132 M-tiles, so the three N-tiles of the
              # dgrad are exactly three full waves (the 8192-row rows above fill 1.3 waves and pay for the tail)
              ("lmhead fwd (engine chunk)", 16896, 50368, 768, 0, 0), ("lmhead dgrad (engine chunk)", 16896, 768, 50368, 0, 1),
              ("lmhead wgrad (engine chunk)", 50368, 768, 16896, 1, 1),
              ("square 8192", 8192, 8192, 8192, 0, 0)]
    for name, M, N, K, amn, bmn in shapes:
        a = torch.randn((K, M) if amn else (M, K), device=dev).to(torch.bfloat16)
        b = torch.randn((K, N) if bmn else (N, K), device=dev).to(torch.bfloat16) * 0.05
        f32 = amn and bmn
        out = torch.empty(M, N, device=dev, dtype=torch.float32 if f32 else torch.bfloat16)
        # weight gradients are timed the way the engine issues them: accumulating into the fp32 bucket (split-K + red.global.add)
        ours = timeit(lambda: ops.gemm(a, b, out, a_mn=bool(amn), b_mn=bool(bmn), epi=ops.EPI_F32 if f32 else ops.EPI_BF16, accumulate=bool(f32)))
        A = a.t() if amn else a
        Bt = b if bmn else b.t()
        if f32:
            cub = timeit(lambda: torch.matmul(A, Bt).float())
        else:
            cub = timeit(lambda: torch.matmul(A, Bt))
        fl = 2.0 * M * N * K
        # same shape on fp8 wgmma (E4M3 x E4M3 forward, E5M2 x E4M3 backward; operands pre-quantised, de-scale in the epilogue)
        a8 = (a.float().clamp(-400, 400)).to(torch.float8_e5m2 if (amn or bmn) else torch.float8_e4m3fn).view(torch.uint8)
        b8 = (b.float().clamp(-400, 400)).to(torch.float8_e4m3fn).view(torch.uint8)
        meta = torch.ones(3, 2, device=dev)
        fp8 = timeit(lambda: ops.gemm_fp8(a8, b8, out, meta, 0, 1, a_mn=bool(amn), b_mn=bool(bmn), epi=ops.EPI_F32 if f32 else ops.EPI_BF16,
                                          a_fmt=ops.E5M2 if (amn or bmn) else ops.E4M3, b_fmt=ops.E4M3, accumulate=bool(f32)))
        mx = None
        if not amn and not bmn and K % 128 == 0:      # block-scaled MXFP8 (forward layout: both operands K-major)
            aq, asf = ops.mx_quantize(a)
            bq, bsf = ops.mx_quantize(b, 2 * ((N + 255) // 256))
            mx = timeit(lambda: ops.gemm_mxfp8(aq, bq, out, asf, bsf))
        rows.append(dict(op=name, M=M, N=N, K=K, ours_ms=ours, cublas_ms=cub, ours_tflops=fl / ours / 1e9, cublas_tflops=fl / cub / 1e9,
                         frac_of_measured_peak=fl / ours / 1e-3 / pk["bf16_flops"], fp8_ms=fp8, fp8_tflops=fl / fp8 / 1e9,
                         fp8_speedup_vs_bf16=ours / fp8, **({"mxfp8_ms": mx, "mxfp8_tflops": fl / mx / 1e9} if mx else {})))
        print(rows[-1], flush=True)
    # memory-bound kernels
    d = 768
    x = torch.randn(T, d, device=dev).to(torch.bfloat16)
    y = torch.empty_like(x)
    g, b_ = torch.ones(d, device=dev), torch.zeros(d, device=dev)
    mean, rstd = torch.empty(T, device=dev), torch.empty(T, device=dev)
    t = timeit(lambda: ops.layernorm_fwd(x, g, b_, y, mean, rstd))
    rows.append(dict(op="layernorm_fwd", ms=t, gbs=2 * x.numel() * 2 / t / 1e6, frac_hbm=2 * x.numel() * 2 / t / 1e-3 / pk["hbm_bytes_per_s"]))
    print(rows[-1])
    tl = timeit(lambda: torch.nn.functional.layer_norm(x, (d,), g.bfloat16(), b_.bfloat16()))
    rows.append(dict(op="layernorm_fwd_torch", ms=tl))
    n = 125_400_000 // 4 * 4
    p, gr, m, v = (torch.randn(n, device=dev) for _ in range(4))
    v.abs_()
    sh = torch.empty(n, device=dev, dtype=torch.bfloat16)
    t = timeit(lambda: ops.ext().fused_optimizer(p, gr, m, v, sh, 0, False, 1e-4, 0.9, 0.9999, 1e-6, 1.0, 3.0, 0.0, 1.0, None))
    rows.append(dict(op="fused_adopt_125M", ms=t, gbs=n * 30 / t / 1e6, frac_hbm=n * 30 / t / 1e-3 / pk["hbm_bytes_per_s"]))
    print(rows[-1])
    lg = torch.randn(4096, 50368, device=dev).to(torch.bfloat16)
    tg = torch.randint(0, 50368, (4096,), device=dev)
    st = torch.zeros(4, dtype=torch.float64, device=dev)
    t = timeit(lambda: ops.cross_entropy(lg, tg, 1e-3, True, st))
    rows.append(dict(op="cross_entropy_4096x50368", ms=t, gbs=lg.numel() * 2 * 3 / t / 1e6))
    print(rows[-1])
    out = Path("gpurun_out")
    out.mkdir(exist_ok=True)
    (out / "bench_kernels.json").write_text(json.dumps(dict(peaks=pk, rows=rows, when=time.time()), indent=1))


if __name__ == "__main__":
    main()
