"""Every GEMM the engine issues in a training step, called the way the engine calls it (same epilogue, operand layout, automatic
cluster choice and output stride), timed with CUDA events and the L2 flushed before each call, as in bench_kernels.py.

    python scripts/gemm_epilogue_bench.py [--tree DIR] [--json FILE]
        MPT-125M at T = 65 536 tokens and its LM-head chunk (16 896 rows), MPT-1B at T = 16 384, amp_bf16 and amp_fp8. Each
        bf16 / E4M3 output GEMM is also timed at K = 768 and K = 3072 with its M, N and epilogue: the time is fitted as
        a + b * K, and `a` is the per-call fixed cost - mostly the epilogue, which a short K cannot hide.
    python scripts/gemm_epilogue_bench.py --save DIR [--tree DIR]
        runs every (A layout, B layout, epilogue, operand type) combination the GEMM accepts, with cluster 1 and 2, on seeded
        inputs and saves D, D2, D8 and the recorded amax, each output embedded in a sentinel-filled wider buffer.
    python scripts/gemm_epilogue_bench.py --compare DIR_A DIR_B
        reports whether two --save runs are bitwise equal (no GPU needed).

--tree imports photon_b200 from another checkout (an older build), so two builds can be compared in one process each."""
import argparse
import json
import statistics
import subprocess
import sys
from pathlib import Path

import torch

ap = argparse.ArgumentParser()
ap.add_argument("--tree", default=str(Path(__file__).resolve().parents[1]))
ap.add_argument("--save", default=None)
ap.add_argument("--compare", nargs=2, default=None)
ap.add_argument("--json", default=None)
ap.add_argument("--iters", type=int, default=20)
args = ap.parse_args()

if args.compare:
    a = torch.load(Path(args.compare[0]) / "outputs.pt")
    b = torch.load(Path(args.compare[1]) / "outputs.pt")
    bad = [k for k in a if k not in b or not torch.equal(a[k], b[k])] + [k for k in b if k not in a]
    print(f"{len(a)} tensors compared, {len(bad)} differ" + "".join(f"\n  differs: {k}" for k in bad))
    sys.exit(1 if bad else 0)

sys.path.insert(0, args.tree)
from photon_b200 import ops  # noqa: E402

assert torch.cuda.is_available(), "this benchmark needs a CUDA device"
dev = torch.device("cuda", 0)
BF = torch.bfloat16


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return {"gpu": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip()}


def rand(*shape, scale=1.0, gen=None):
    return (torch.randn(*shape, device=dev, generator=gen) * scale).to(BF)


def q8(x, fmt):
    return x.float().to(torch.float8_e5m2 if fmt == ops.E5M2 else torch.float8_e4m3fn).view(torch.uint8)


def make_call(M, N, K, epi, a_mn=False, b_mn=False, fp8=False, bias=True, gen=None, out_pad=0, out_off=0, cluster=0):
    """The GEMM `epilogue(A @ B^T)` with freshly made operands; returns (call, outputs). Outputs other than fp32 sit at column
    `out_off` of buffers `out_pad` columns wider (and 8 rows taller) than [M, N], pre-filled with a sentinel."""
    a_fmt = ops.E5M2 if (a_mn or b_mn) else ops.E4M3            # the engine's backward GEMMs read E5M2 gradients
    a = rand(*((K, M) if a_mn else (M, K)), gen=gen)
    b = rand(*((K, N) if b_mn else (N, K)), scale=0.05, gen=gen)
    if fp8:
        a, b = q8(a, a_fmt), q8(b, ops.E4M3)
    f32 = epi == ops.EPI_F32
    two = epi in (ops.EPI_GELU_DUAL, ops.EPI_GELU_GRAD, ops.EPI_GELU_GRAD_Q8)

    def out_buf(dtype):
        if f32 or out_pad == 0:
            return torch.zeros(M, N, device=dev, dtype=dtype) if f32 else torch.empty(M, N, device=dev, dtype=dtype)
        buf = torch.full((M + 8, N + out_pad), 3, device=dev, dtype=torch.uint8).view(dtype) if dtype == torch.uint8 else \
            torch.full((M + 8, N + out_pad), -7.0, device=dev, dtype=dtype)
        return buf, buf[:M, out_off:out_off + N]

    outs = {}
    d = out_buf(torch.float32 if f32 else BF)
    if isinstance(d, tuple):
        outs["D"], d = d
    else:
        outs["D"] = d
    kw = dict(a_mn=a_mn, b_mn=b_mn, epi=epi, cluster=cluster)
    if bias and not f32:
        kw["bias"] = torch.randn(N, device=dev, generator=gen) * 0.1
    if epi in (ops.EPI_RESIDUAL, ops.EPI_DGELU, ops.EPI_MUL):
        kw["aux"] = rand(M, N, gen=gen)
    if two:
        d2 = out_buf(BF)
        if isinstance(d2, tuple):
            outs["D2"], d2 = d2
        else:
            outs["D2"] = d2
        kw["out2"] = d2
    if f32:
        kw["accumulate"] = True
    if not fp8:
        return (lambda: ops.gemm(a, b, d, **kw)), outs
    meta = torch.ones(3, 3, device=dev)
    meta[0, 2], meta[1, 2], meta[2, 2] = 16.0, 1 / 16.0, 0.0     # role 2: the E4M3 output of the Q8 epilogue
    kw.update(a_fmt=a_fmt, b_fmt=ops.E4M3)
    if epi == ops.EPI_GELU_GRAD_Q8:
        d8 = out_buf(torch.uint8)
        if isinstance(d8, tuple):
            outs["D8"], d8 = d8
        else:
            outs["D8"] = d8
        kw.update(out8=d8, role_out=2)
        d = kw["out2"]                   # the engine passes the gelu' buffer as the unused primary output
        outs.pop("D")
        outs["amax"] = meta[2]
    return (lambda: ops.gemm_fp8(a, b, d, meta, 0, 1, **kw)), outs


flush = None


def timeit(fn, iters, warm=3):
    global flush
    if flush is None:
        flush = torch.empty(256 * 1024 * 1024, dtype=torch.uint8, device=dev)
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
        ts.append(s.elapsed_time(e) * 1e3)
    return statistics.median(ts)


def engine_gemms(d, T, V, chunk):
    """(name, M, N, K, epi, a_mn, b_mn, bias) of one microbatch's block GEMMs (one layer) and LM-head chunk, in engine order."""
    E = ops
    return [
        ("qkv fwd", T, 3 * d, d, E.EPI_BF16, 0, 0, 1), ("out fwd", T, d, d, E.EPI_RESIDUAL, 0, 0, 1),
        ("up fwd", T, 4 * d, d, E.EPI_GELU_GRAD, 0, 0, 1), ("down fwd", T, d, 4 * d, E.EPI_RESIDUAL, 0, 0, 1),
        ("head fwd", chunk, V, d, E.EPI_BF16, 0, 0, 0), ("head dgrad", chunk, d, V, E.EPI_BF16, 0, 1, 0),
        ("head wgrad", V, d, chunk, E.EPI_F32, 1, 1, 0),
        ("down wgrad", d, 4 * d, T, E.EPI_F32, 1, 1, 0), ("down dgrad", T, 4 * d, d, E.EPI_MUL, 0, 1, 0),
        ("up wgrad", 4 * d, d, T, E.EPI_F32, 1, 1, 0), ("up dgrad", T, d, 4 * d, E.EPI_BF16, 0, 1, 0),
        ("out wgrad", d, d, T, E.EPI_F32, 1, 1, 0), ("out dgrad", T, d, d, E.EPI_BF16, 0, 1, 0),
        ("qkv wgrad", 3 * d, d, T, E.EPI_F32, 1, 1, 0), ("qkv dgrad", T, d, 3 * d, E.EPI_BF16, 0, 1, 0),
    ]


def bench():
    info = gpu_info()
    print(json.dumps(info), flush=True)
    rows = []
    models = [("mpt-125m", 768, 65536, 50368, 16896), ("mpt-1b", 2048, 16384, 50368, 16384)]
    for model, d, T, V, chunk in models:
        for prec in ("amp_bf16", "amp_fp8"):
            fp8 = prec == "amp_fp8"
            for name, M, N, K, epi, amn, bmn, bias in engine_gemms(d, T, V, chunk):
                if fp8 and name.startswith("head"):
                    continue                    # the LM head runs in bf16 under amp_fp8 as well
                e = ops.EPI_GELU_GRAD_Q8 if fp8 and epi == ops.EPI_GELU_GRAD else epi
                call, _ = make_call(M, N, K, e, bool(amn), bool(bmn), fp8, bool(bias))
                us = timeit(call, args.iters)
                row = dict(model=model, prec=prec, op=name, M=M, N=N, K=K, epi=e, us=round(us, 1), tflops=round(2 * M * N * K / us / 1e6, 1))
                if epi != ops.EPI_F32:
                    # the same M, N and epilogue at K = 768 and 3072: t = a + b K
                    t = {}
                    for k in (768, 3072):
                        c, _ = make_call(M, N, k, e, bool(amn), bool(bmn), fp8, bool(bias))
                        t[k] = timeit(c, args.iters)
                        del c
                    slope = (t[3072] - t[768]) / (3072 - 768)
                    fixed = t[768] - 768 * slope
                    row.update(us_k768=round(t[768], 1), us_k3072=round(t[3072], 1), fixed_us=round(fixed, 1),
                               fixed_share_k768=round(fixed / t[768], 3))
                rows.append(row)
                print(json.dumps(row), flush=True)
                del call
                torch.cuda.empty_cache()
    if args.json:
        Path(args.json).parent.mkdir(parents=True, exist_ok=True)
        Path(args.json).write_text(json.dumps(dict(info=info, tree=args.tree, rows=rows), indent=1))


# every (a_mn, b_mn, epilogue, fp8) the GEMM accepts
CASES = [(0, 0, 0, 0), (0, 0, 1, 0), (0, 0, 2, 0), (0, 0, 4, 0), (0, 1, 0, 0), (0, 1, 3, 0), (0, 1, 6, 0), (0, 0, 5, 0), (0, 1, 4, 0),
         (1, 1, 4, 0), (1, 1, 0, 0), (1, 0, 4, 0), (1, 0, 0, 0),
         (0, 0, 0, 1), (0, 0, 1, 1), (0, 0, 5, 1), (0, 0, 7, 1), (0, 0, 4, 1), (0, 0, 6, 1)]


def save(out_dir):
    res = {}
    # M tail with an odd M-tile count, N % 64 != 0, K tails (bf16 and fp8 k-blocks); then an engine-sized block GEMM
    for M, N, K in ((520, 328, 208), (72, 584, 144), (2048, 3072, 768)):
        for amn, bmn, epi, fp8 in CASES:
            n = N + 8 if epi == ops.EPI_GELU_GRAD_Q8 and N % 16 else N     # E4M3 rows are whole 16-byte pieces
            for cl in (1, 2):
                gen = torch.Generator(device=dev)
                gen.manual_seed(1234)
                call, outs = make_call(M, n, K, epi, bool(amn), bool(bmn), bool(fp8), True, gen=gen, out_pad=64 - n % 16, out_off=32, cluster=cl)
                call()
                torch.cuda.synchronize()
                for k, v in outs.items():
                    res[f"M{M}_N{n}_K{K}_a{amn}_b{bmn}_epi{epi}_fp8{fp8}_cl{cl}_{k}"] = v.detach().cpu().clone()
    Path(out_dir).mkdir(parents=True, exist_ok=True)
    torch.save(res, Path(out_dir) / "outputs.pt")
    print(f"saved {len(res)} tensors to {out_dir}")


if __name__ == "__main__":
    if args.save:
        save(args.save)
    else:
        bench()
