"""PascoNet.step — Net.step(batch, "train") on the engine — with and without the per-step evaluation of subnets 0 and
M − 1 (predict.evaluate_step: step_entries + metrics.Evaluator(uncertainty=False)).

    python tools/step_eval_bench.py [--subnets 1 2] [--steps 5] [--warmup 2]

Scene 256x256x32 @10 %, f = 64, Q = 100, ten masks.  Per M, one JSON line with, for each arm: the step (forward,
fused_training_loss, backward, fused AdamW) median and range over --steps steps, the arms alternated step by step, and
the step's peak memory; the evaluation alone on one forward output (bracketed by synchronises, median over --steps
calls); its host syncs, kernel launches and peak memory (evaluate_hook_bench.counted); and the evaluated subnets' PQ /
mIoU after the timed steps, so that a run shows the metrics are live.  The card's name and power limit are read in the
same process.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools")]
from evaluate_hook_bench import counted  # noqa: E402
from infer_bench import gpu_state  # noqa: E402

GRID, OCC, IN_CH, K = (256, 256, 32), 0.10, 283, 20


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("step_eval_bench.py: no CUDA device")
    from pasco_b200 import _lib
    from pasco_b200 import criterion as CR
    from pasco_b200 import metrics as MT
    from pasco_b200 import predict as PR
    from pasco_b200.net3d import PascoNet, evaluated_subnets
    from pasco_b200.synthetic import make_scene, training_batch
    _lib.load()
    dev = torch.device("cuda")
    for M in a.subnets:
        torch.manual_seed(0)
        net = PascoNet(n_classes=K, n_infers=M, in_channels=IN_CH, f=64, num_queries=100).to(dev).train()
        opt = torch.optim.AdamW([p for p in net.parameters() if p.requires_grad], lr=1e-4, weight_decay=1e-4, fused=True)
        sc = training_batch(make_scene(GRID, OCC, M, IN_CH, K, seed=0, n_masks=10))
        sc = dict(sc, in_feats=[f.to(dev) for f in sc["in_feats"]], in_coords=[c.to(dev) for c in sc["in_coords"]])
        crit = CR.SetCriterion(K, [torch.ones(K + 1, device=dev)] * M, torch.ones(K, device=dev))
        subnets = evaluated_subnets(M)
        evs = {i: MT.Evaluator(n_entries=1, n_classes=K, uncertainty=False) for i in subnets}
        arms = {"without_metrics": None, "with_metrics": evs}

        def step(metrics):
            opt.zero_grad(set_to_none=True)
            total, _ = net.step(sc, crit, net.class_frequencies, metrics=metrics)
            total.backward()
            opt.step()
        times, peaks = {k: [] for k in arms}, {}
        for i in range(a.warmup + a.steps):
            for name, metrics in arms.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                step(metrics)
                torch.cuda.synchronize()
                if i >= a.warmup:
                    times[name].append((time.perf_counter() - t0) * 1e3)
        for name, metrics in arms.items():
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            step(metrics)
            torch.cuda.synchronize()
            peaks[name] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
        res = {"M": M, "scene": f"{GRID[0]}x{GRID[1]}x{GRID[2]} @{OCC:.0%}", "f": 64, "Q": 100, "masks": 10,
               "evaluated_subnets": subnets}
        for name, ts in times.items():
            res[name] = dict(step_ms_median=round(statistics.median(ts), 1), step_ms_range=[round(min(ts), 1),
                             round(max(ts), 1)], step_peak_gib=peaks[name])
        res["metrics_after_steps"] = {i: {"All_pq": round(d["All"]["pq"], 4), "mIoU": round(d["iou_ssc_mean"], 4),
                                          "IoU": round(d["iou"], 4)} for i, d in
                                      ((i, ev.compute()[0]) for i, ev in evs.items())}
        with torch.no_grad():
            out = net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
        scratch = {i: MT.Evaluator(n_entries=1, n_classes=K, uncertainty=False) for i in subnets}
        ev_ms = []
        for _ in range(a.steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            PR.evaluate_step(out, sc, scratch)
            torch.cuda.synchronize()
            ev_ms.append((time.perf_counter() - t0) * 1e3)
        res["evaluation"] = dict(ms_median=round(statistics.median(ev_ms), 2), ms_range=[round(min(ev_ms), 2),
                                 round(max(ev_ms), 2)], stated_syncs=len(subnets) * (PR.STEP_ENTRY_SYNCS +
                                                                                      MT.VAL_UPDATE_SYNCS),
                                 **counted(lambda: PR.evaluate_step(out, sc, scratch)))
        import warnings
        with warnings.catch_warnings(record=True) as w:                 # where the evaluation's host syncs are
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                PR.evaluate_step(out, sc, scratch)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        res["evaluation"]["sync_sites"] = [f"{os.path.basename(x.filename)}:{x.lineno}" for x in w
                                           if "synchroniz" in str(x.message)]
        res["gpu"] = gpu_state()
        print(json.dumps(res), flush=True)
        del net, opt, out
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
