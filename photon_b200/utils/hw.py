"""Hardware constants and roofline denominators of the target GPU, the NVIDIA H100 SXM (80 GB HBM3)."""
from __future__ import annotations

import json
from functools import lru_cache
from pathlib import Path

NUM_SMS = 132
L2_BYTES = 50 * 1024 * 1024
# NVIDIA data-sheet figures of the H100 SXM (700 W), used only when MEASURED_PEAKS.json is absent; they are upper bounds, not
# measurements: a card with a lower power limit sustains less
FALLBACK_HBM_GBS = 3350.0
FALLBACK_BF16_TFLOPS = 989.0
NVLINK_PEER_GBS = 450.0        # NVLink 4: 900 GB/s bidirectional per GPU, i.e. 450 GB/s per direction (data sheet)
NVLINK_ALLREDUCE_BUS_GBS = 450.0


@lru_cache(maxsize=1)
def measured_peaks() -> dict[str, float]:
    root = Path(__file__).resolve().parents[2]
    p = root / "MEASURED_PEAKS.json"
    out = {"hbm_bytes_per_s": FALLBACK_HBM_GBS * 1e9, "bf16_flops": FALLBACK_BF16_TFLOPS * 1e12,
           "bf16_flops_sustained": FALLBACK_BF16_TFLOPS * 1e12, "source": "fallback"}
    if p.exists():
        try:
            d = json.loads(p.read_text())
            out = {"hbm_bytes_per_s": float(d["hbm_gbs"]) * 1e9, "bf16_flops": float(d["bf16_tflops"]) * 1e12,
                   "bf16_flops_sustained": float(d.get("bf16_tflops_sustained", d["bf16_tflops"])) * 1e12,
                   "source": "measured"}
        except Exception:  # noqa: BLE001
            pass
    return out
