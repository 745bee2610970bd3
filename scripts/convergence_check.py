"""Short flagship-shape training run on ONE GPU: MPT-125M, 2 clients x 24 local steps x 3 rounds, batch 16 x 2048, on a
LEARNABLE synthetic stream (each sequence repeats a short random motif), engine kernels vs the stock PyTorch backend from
the same initial weights. Prints the per-round loss of both; the curves must fall together.
Run on a GPU box:  python scripts/convergence_check.py
"""
import json
import sys

import torch

sys.path.insert(0, ".")
from photon_b200.models.mpt import MPTConfig  # noqa: E402
from photon_b200.train.trainer import Trainer  # noqa: E402


def make_batches(n, b, S, vocab, seed):
    g = torch.Generator().manual_seed(seed)
    out = []
    for _ in range(n):
        motif = torch.randint(0, vocab, (b, 64), generator=g)
        ids = motif.repeat(1, S // 64)
        noise = torch.rand(b, S, generator=g) < 0.05
        ids = torch.where(noise, torch.randint(0, vocab, (b, S), generator=g), ids)
        out.append(ids)
    return out


def run(kernels, batches, steps, precision="amp_bf16", lr=6e-4):
    cfg = MPTConfig()   # MPT-125M
    dev = torch.device("cuda", 0)

    class Loader:
        def __iter__(self):
            i = 0
            while True:
                yield {"input_ids": batches[i % len(batches)].pin_memory()}
                i += 1

    tr = Trainer(cfg, optimizer_cfg=dict(name="adopt", lr=lr, betas=[0.9, 0.9999], eps=1e-6, weight_decay=0.0),
                 scheduler_cfg=dict(name="cosine_with_warmup", t_warmup="10ba", t_max=f"{steps}ba", alpha_f=0.1), train_loader=Loader(),
                 global_train_batch_size=16, device_train_microbatch_size=16, precision=precision, max_duration=f"{steps}ba",
                 grad_clip_norm=1.0, device=dev, kernels=kernels, seed=17)
    tr.fit(f"{steps}ba")
    losses = [float(v) for _, v in tr.loggers[0].data["loss/train/total"]]
    kind = tr.state.backend.kind
    tr.close()
    return kind, losses


def fp8_parity():
    """amp_fp8 engine (fp8 wgmma GEMMs) vs the bf16 engine: 60 steps from the same weights on the same data, at a
    learning rate high enough for the loss to move (3e-3): the two curves must fall together."""
    steps = 60
    batches = make_batches(steps, 16, 2048, 50368, seed=5)
    res = {}
    for name, prec in (("engine_bf16", "amp_bf16"), ("engine_fp8", "amp_fp8")):
        kind, losses = run({}, batches, steps, precision=prec, lr=3e-3)
        res[name] = {"backend": kind, "precision": prec, "loss_first": losses[0], "loss_step10": losses[9], "loss_step20": losses[19],
                     "loss_step30": losses[29], "loss_step45": losses[44], "loss_last": losses[-1]}
        print(name, json.dumps(res[name]), flush=True)
    gap = max(abs(res["engine_fp8"][k] - res["engine_bf16"][k]) for k in res["engine_bf16"] if k.startswith("loss"))
    fell = res["engine_bf16"]["loss_first"] - res["engine_bf16"]["loss_last"]
    print(json.dumps({"max_loss_gap_fp8_vs_bf16": gap, "bf16_loss_drop": fell, "ok": bool(gap < 0.05 + 0.05 * fell and res["engine_fp8"]["loss_last"] < res["engine_fp8"]["loss_first"])}))


def main():
    if len(sys.argv) > 1 and sys.argv[1] == "fp8":
        fp8_parity()
        return
    steps = 60
    batches = make_batches(steps, 16, 2048, 50368, seed=5)
    res = {}
    for name, kernels in (("b200", {}), ("torch", dict(gemm="torch", attention="torch", norm="torch", loss="torch", optimizer="torch"))):
        kind, losses = run(kernels, batches, steps)
        res[name] = {"backend": kind, "loss_first": losses[0], "loss_step10": losses[9], "loss_step30": losses[29], "loss_last": losses[-1]}
        print(name, json.dumps(res[name]), flush=True)
    d = abs(res["b200"]["loss_last"] - res["torch"]["loss_last"])
    assert res["b200"]["loss_last"] < res["b200"]["loss_step30"] < res["b200"]["loss_first"], "engine loss is not falling"
    print(json.dumps({"final_loss_gap": d, "ok": bool(d < 0.05)}))


if __name__ == "__main__":
    main()
