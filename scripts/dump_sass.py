"""Per-kernel SASS listings of the flagship sm_90a kernels -> profiles/sass/*.sass (not tracked), plus the mnemonic census.

Needs no GPU (cuobjdump reads the cross-compiled objects under build/obj). One listing per kernel family; the Hopper
instructions each one is built on are counted at the top of every file: HGMMA / QGMMA (wgmma on bf16 / fp8 operands),
UTMALDG / UTMASTG / UTMAREDG (TMA load / store / reduce), UBLKCP (bulk copy), SYNCS (mbarrier), USETMAXREG (setmaxnreg),
REDG (global reductions), *MULTIMEM* / *MC forms (multimem.ld_reduce / multimem.st).
"""
from __future__ import annotations

import re
import subprocess
import sys
from collections import Counter
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
OBJ = ROOT / "build" / "obj"
OUT = ROOT / "profiles" / "sass"

# (object file, regex on the demangled kernel name, output name)
PICKS = [
    ("gemm_tcgen05.cu.o", r"gemm_kernel<0, 0, 1, 2, 0>", "gemm_bf16_fwd_residual_2cta"),
    ("gemm_tcgen05.cu.o", r"gemm_kernel<1, 1, 4, 2, 0>", "gemm_bf16_wgrad_f32_2cta"),
    ("gemm_tcgen05.cu.o", r"gemm_kernel<0, 0, 7, 2, 1>", "gemm_fp8_fwd_gelu_q8_2cta"),
    ("gemm_tcgen05.cu.o", r"gemm_kernel<0, 0, 6, 2, 1>", "gemm_fp8_dgrad_mul_2cta"),
    ("gemm_tcgen05.cu.o", r"gemm_kernel<0, 0, 4, 2, 1>", "gemm_fp8_wgrad_f32_2cta"),
    ("gemm_tcgen05.cu.o", r"transpose_u8_kernel", "transpose_u8"),
    ("gemm_mxfp8.cu.o", r"gemm_mx_kernel", "gemm_mxfp8_block_scaled"),
    ("gemm_mxfp8.cu.o", r"mx_quantize_kernel", "mx_quantize"),
    ("attention_tcgen05.cu.o", r"attn_fwd_kernel<64", "attention_fwd_d64"),
    ("attention_tcgen05.cu.o", r"attn_bwd_kernel<64", "attention_bwd_d64"),
    ("attention_tcgen05.cu.o", r"attn_fwd_kernel<128", "attention_fwd_d128"),
    ("comm.cu.o", r"fed_round_kernel", "fed_round"),
    ("comm.cu.o", r"ddp_allreduce_kernel", "ddp_allreduce"),
    ("comm.cu.o", r"ddp_zero_step_kernel", "ddp_zero_step"),
    ("comm.cu.o", r"zero3_reduce_kernel", "zero3_reduce"),
    ("fp8_ops.cu.o", r"ln_fwd_q8_kernel<3, false>", "layernorm_fwd_q8_d768"),
    ("fp8_ops.cu.o", r"colsum_quant_kernel<1>", "colsum_quant_e5m2"),
    ("fused_ops.cu.o", r"optim_kernel", "fused_optimizer"),
    ("fused_ops.cu.o", r"ce_kernel", "cross_entropy"),
]
KEY = re.compile(r"\b(HGMMA(?:\.[A-Z0-9_]+)*|QGMMA(?:\.[A-Z0-9_]+)*|UTMA[A-Z]+(?:\.[A-Z0-9_]+)*|UBLKCP(?:\.[A-Z0-9_]+)*|SYNCS(?:\.[A-Z0-9_]+)*|"
                 r"USETMAXREG(?:\.[A-Z0-9_]+)*|REDG(?:\.[A-Z0-9_]+)*|[A-Z]*MULTIMEM[A-Z.0-9_]*|LDGMC[A-Z.0-9_]*|REDG?MC[A-Z.0-9_]*|STGMC[A-Z.0-9_]*|"
                 r"HMMA[.A-Z0-9_]*|F2FP[.A-Z0-9_]*)")


def sass_functions(obj: Path) -> dict[str, str]:
    txt = subprocess.run(["cuobjdump", "-sass", str(obj)], capture_output=True, text=True, check=True).stdout
    parts = re.split(r"\n\s*Function : ", txt)
    out = {}
    for p in parts[1:]:
        name, _, body = p.partition("\n")
        out[name.strip()] = body
    return out


def demangle(names: list[str]) -> dict[str, str]:
    r = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True)
    return dict(zip(names, r.stdout.splitlines())) if r.returncode == 0 else {n: n for n in names}


def main() -> None:
    OUT.mkdir(parents=True, exist_ok=True)
    census = []
    cache: dict[str, tuple[dict[str, str], dict[str, str]]] = {}
    for obj, pat, outname in PICKS:
        if obj not in cache:
            fns = sass_functions(OBJ / obj)
            cache[obj] = (fns, demangle(list(fns)))
        fns, dm = cache[obj]
        hit = [m for m in fns if re.search(pat, dm[m])]
        if not hit:
            print(f"[dump_sass] no kernel matches {pat} in {obj}", file=sys.stderr)
            continue
        body = fns[hit[0]]
        cnt = Counter(KEY.findall(body))
        n_instr = len(re.findall(r"/\*[0-9a-f]{4}\*/", body))
        head = [f"// {dm[hit[0]]}", f"// object: build/obj/{obj}   (nvcc -gencode arch=compute_90a,code=sm_90a -lineinfo -O3)",
                f"// {n_instr} SASS instructions; Hopper tensor-core / TMA / barrier / reduction mnemonics: " + (", ".join(f"{k} x{v}" for k, v in sorted(cnt.items())) or "none")]
        # keep the instruction text only (drop the encoding words): small, diff-able files
        lines = [re.sub(r"\s*/\* 0x[0-9a-f]{16} \*/\s*$", "", ln) for ln in body.splitlines() if not re.match(r"^\s*/\* 0x[0-9a-f]{16} \*/\s*$", ln)]
        (OUT / f"{outname}.sass").write_text("\n".join(head) + "\n" + "\n".join(lines) + "\n")
        census.append(f"{outname:32s} {n_instr:6d} instr  " + " ".join(f"{k}={v}" for k, v in sorted(cnt.items())))
    (OUT / "README.txt").write_text("Per-kernel SASS (scripts/dump_sass.py). Mnemonic census:\n\n" + "\n".join(census) + "\n")
    print("\n".join(census))


if __name__ == "__main__":
    main()
