"""Registers / spills / shared memory of every kernel, from the `-Xptxas -v` logs of the last build (build/obj/*.log) ->
profiles/ptxas_summary.txt. Runs on the CPU box; names are demangled with c++filt."""
from __future__ import annotations

import re
import subprocess
from pathlib import Path

ROOT = Path(__file__).resolve().parents[1]
PAT = re.compile(r"Compiling entry function '(\S+)' for 'sm_90a'.*?\n(?:.*?\n)??\s*(\d+) bytes stack frame, (\d+) bytes spill stores, (\d+) bytes spill loads\n"
                 r".*?Used (\d+) registers(?:, used (\d+) barriers)?(?:, (\d+) bytes smem)?", re.S)


def main() -> None:
    rows = []
    for log in sorted((ROOT / "build" / "obj").glob("*.log")):
        txt = log.read_text()
        for m in PAT.finditer(txt):
            rows.append((log.name.replace(".cu.log", ""), m.group(1), int(m.group(5)), int(m.group(2)), int(m.group(3)), int(m.group(4)),
                         int(m.group(7) or 0)))
    names = [r[1] for r in rows]
    dem = subprocess.run(["c++filt"], input="\n".join(names), capture_output=True, text=True).stdout.splitlines() if names else []
    out = ["# ptxas -v summary of the sm_90a build (scripts/ptxas_summary.py): registers/thread, stack frame, spill stores/loads (bytes), static smem",
           "# (dynamic shared memory is requested at launch: see the *Cfg::SMEM constants in csrc/)", ""]
    for (unit, _raw, regs, stack, st, ld, smem), name in zip(rows, dem):
        short = name.replace("pb::(anonymous namespace)::", "").replace("(anonymous namespace)::", "").replace("void ", "")
        short = re.sub(r"\((?!anonymous).*", "", short)
        out.append(f"{unit:22s} {regs:4d} regs  stack {stack:5d}  spill {st:5d}/{ld:5d}  smem {smem:6d}  {short[:110]}")
    spilled = sum(1 for r in rows if r[4] or r[5])
    out += ["", f"{len(rows)} kernels, {spilled} with spills"]
    (ROOT / "profiles" / "ptxas_summary.txt").write_text("\n".join(out) + "\n")
    print("\n".join(out[-12:]))


if __name__ == "__main__":
    main()
