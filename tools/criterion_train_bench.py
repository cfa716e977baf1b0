"""A PascoNet training step on three losses: the compact `losses.total_loss`, the reference restatement
`criterion.training_loss` on the device, and `criterion.fused_training_loss` on the grouped setloss kernels.

    python tools/criterion_train_bench.py [--subnets 1 2] [--steps 5] [--warmup 2]

Scene 256x256x32 @10 %, f = 64, Q = 100, ten masks.  Per M, one JSON line with, for each arm: the step (forward, loss,
backward, fused AdamW) median and range over --steps steps, the arms alternated step by step; the loss's forward time
alone (bracketed by synchronises, a separate pass); host syncs, kernel launches and peak memory of one loss call
(evaluate_hook_bench.counted); and from a torch.profiler pass of the fused arm, each setloss kernel's time against the
bytes it must move (must_read) at 3.35 TB/s.  The card's
name and power limit are read in the same process.  Writes nothing.
"""
import argparse
import json
import os
import re
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
from evaluate_hook_bench import counted  # noqa: E402
from infer_bench import gpu_state  # noqa: E402

GRID, OCC, IN_CH, K = (256, 256, 32), 0.10, 283, 20
HBM = 3.35e12           # H100 SXM HBM3 bytes/s (data sheet)


def must_read(out, K):
    """Bytes each setloss kernel of one fused_training_loss forward must move at least, from the forward output: the
    matcher cost reads every level's fp32 logits [N, Q] once; the pair sums read the matched columns [N, P ≤ T]; the
    ssc forward reads the kept columns [N, kq] and writes [N, K]; the Lovász errors read [P, C] logits and write the
    probabilities and errors; the Lovász grad reads the sorted errors, the permutation (int64) and the gathered labels
    and writes the grad, each [C, P]."""
    cost = pairs = ssc = lov_rows = 0
    T = 10
    for p in out["panop_predictions"]:
        for i, lv in enumerate([p] + p["aux_outputs"]):
            N, Q = lv["voxel_logits"].F.shape
            cost += N * Q * 4 + N * 5
            pairs += N * min(Q, T) * 4 + N * 5
            if i:
                kq = int((lv["query_logits"][0].argmax(-1) != K).sum())
                if kq:
                    ssc += N * (kq + K) * 4
                    lov_rows += N * K
    for per in out["sem_logits_at_scales"].values():
        for sl in per:
            lov_rows += sl.F.numel()
    return {"k_sl_cost": cost, "k_sl_pair_sums": pairs, "k_sl_ssc_forward": ssc, "k_lov_errors": lov_rows * 12,
            "k_lov_grad": lov_rows * 20}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("criterion_train_bench.py: no CUDA device")
    from pasco_b200 import _lib, ops
    from pasco_b200 import criterion as CR
    from pasco_b200.losses import total_loss
    from pasco_b200.net3d import PascoNet
    from pasco_b200.synthetic import make_scene, training_batch
    _lib.load()
    dev = torch.device("cuda")
    for M in a.subnets:
        torch.manual_seed(0)
        net = PascoNet(n_classes=K, n_infers=M, in_channels=IN_CH, f=64, num_queries=100).to(dev).train()
        params = [p for p in net.parameters() if p.requires_grad]
        opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-4, fused=True)
        sc = training_batch(make_scene(GRID, OCC, M, IN_CH, K, seed=0, n_masks=10))
        args = ([f.to(dev) for f in sc["in_feats"]], [c.to(dev) for c in sc["in_coords"]], sc["global_min_Cs"],
                sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
        crit = CR.SetCriterion(K, [torch.ones(K + 1, device=dev)] * M, torch.ones(K, device=dev))
        losses = {"total_loss": lambda out: total_loss(out, sc, K, net.class_frequencies),
                  "training_loss": lambda out: CR.training_loss(out, sc, crit, net.class_frequencies)[0],
                  "fused_training_loss": lambda out: CR.fused_training_loss(out, sc, crit, net.class_frequencies)[0]}

        def step(name):
            opt.zero_grad(set_to_none=True)
            losses[name](net(*args)).backward()
            opt.step()
        times = {k: [] for k in losses}
        for i in range(a.warmup + a.steps):
            for name in losses:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                step(name)
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[name].append((time.perf_counter() - t0) * 1e3)
        res = {"M": M, "scene": f"{GRID[0]}x{GRID[1]}x{GRID[2]} @{OCC:.0%}", "f": 64, "Q": 100, "masks": 10}
        with torch.no_grad():
            out = net(*args)
        for name, fn in losses.items():
            fwd = []
            for _ in range(a.steps):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fn(out)
                torch.cuda.synchronize()
                fwd.append((time.perf_counter() - t0) * 1e3)
            ts = times[name]
            res[name] = dict(step_ms_median=round(statistics.median(ts), 1), step_ms_range=[round(min(ts), 1),
                             round(max(ts), 1)], loss_forward_ms=round(statistics.median(fwd), 2), **counted(lambda: fn(out)))
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as p:
            losses["fused_training_loss"](out)
            torch.cuda.synchronize()
        kern = {}
        for ev in p.key_averages():
            m = re.search(r"\b(k_sl_\w+|k_lov_\w+)", ev.key)
            if m:
                kern[m.group(1)] = round(kern.get(m.group(1), 0.0) + ev.device_time_total / 1e3, 3)
        res["fused_setloss_kernels_ms"] = kern
        res["fused_setloss_bytes_vs_hbm"] = {k: dict(mb=round(v / 1e6, 1), ms=kern.get(k),
                                                     hbm_frac=round(v / HBM / (kern[k] / 1e3), 3) if kern.get(k) else None)
                                             for k, v in must_read(out, K).items()}
        res["gpu"] = gpu_state()
        print(json.dumps(res), flush=True)
        del net, opt, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
