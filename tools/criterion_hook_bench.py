"""Net.step(batch, "train") plus backward of the UNMODIFIED reference on the drop-in, with the criterion hook off and on
(pasco_b200/hooks.py install(criterion=True)); the attention, post-processing and evaluation hooks are on in both modes.

    python tools/criterion_hook_bench.py [--subnets 1 2] [--steps 8] [--warmup 1]

Workload: tools/dropin_scale_bench.py's training batch at 256x256x32 @10 % (f = 64, Q = 100, recipe-calibrated random
weights, ten box masks, dense semantic labels, per-subnet class weights on the host as the reference keeps them),
criterion off and on alternated step by step.  Per mode:
  * the step's median and range in ms (host clock, ended by a device synchronise);
  * the criterion's own forward time per step: every SetCriterion.forward and completion-loss call bracketed by
    device synchronises, in a separate pass (the criterion's backward runs inside loss.backward() and is not separated);
  * host synchronisations (torch.cuda.set_sync_debug_mode), kernel launches (torch.profiler) and peak memory;
  * the ten kernels with the most CUDA time, and every setloss.cu kernel, in a separate torch.profiler pass;
  * the bytes the match-cost kernel must read (4·N·Q + 4·N·⌈T/32⌉ per level) against 3.35 TB/s, with its measured time.
Prints one JSON line per subnet count, with the card's name and power limit read in the same run; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle", "_ref"), os.path.join(ROOT, "compat"),
                os.path.join(ROOT, "tests", "golden")]
from evaluate_hook_bench import counted, stats, timed  # noqa: E402
from infer_bench import GRID, gpu_state  # noqa: E402
from postprocess_bench import reference_net  # noqa: E402

HBM_BYTES_PER_S = 3.35e12


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=on)


def criterion_time(net, one, steps):
    """ms per step inside SetCriterion.forward and the completion loss, each call bracketed by device synchronises;
    also the rows, queries and targets of every level the matcher saw."""
    import pasco.models.net_panoptic_sparse as nps
    from pasco.loss.criterion_sparse import SetCriterion
    spent, shapes = [0.0], []
    fwd, compl = SetCriterion.forward, nps.compute_sem_compl_loss

    def wrap(fn):
        def inner(*a, **k):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            out = fn(*a, **k)
            torch.cuda.synchronize()
            spent[0] += time.perf_counter() - t0
            return out
        return inner

    def fwd_rec(self, sem, outputs, targets, *a, **k):
        for lv in [outputs] + list(outputs.get("aux_outputs", [])):
            shapes.append((lv["voxel_logits"].F.shape[0], lv["voxel_logits"].F.shape[1], targets[0]["masks"].shape[0]))
        return fwd(self, sem, outputs, targets, *a, **k)

    SetCriterion.forward = wrap(fwd_rec)
    nps.compute_sem_compl_loss = wrap(compl)
    try:
        per = []
        for _ in range(steps):
            spent[0] = 0.0
            shapes.clear()
            one()
            per.append(spent[0] * 1e3)
    finally:
        SetCriterion.forward, nps.compute_sem_compl_loss = fwd, compl
    return {"criterion_forward_ms_per_step_median": round(statistics.median(per), 1)}, list(shapes)


def kernel_table(one):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        one()
        torch.cuda.synchronize()
    agg = {}
    for ev in p.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA:
            n, t = agg.get(ev.name, (0, 0.0))
            agg[ev.name] = (n + 1, t + ev.device_time_total / 1e3)
    top = sorted(agg.items(), key=lambda kv: -kv[1][1])[:10]
    ours = sorted((kv for kv in agg.items() if "k_sl_" in kv[0] or "k_lov_" in kv[0]), key=lambda kv: -kv[1][1])
    cost = [v for k, v in agg.items() if "k_sl_cost" in k and "finish" not in k]
    row = lambda k, n, t: {"kernel": k[:90], "calls": n, "ms": round(t, 3)}  # noqa: E731
    return ([row(k, n, t) for k, (n, t) in top], [row(k, n, t) for k, (n, t) in ours], cost[0] if cost else None)


def run(M, a, hooks, make_scene):
    from dropin_scale_bench import train_batch
    net = reference_net(M).train()
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1) for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K, device="cuda")
    net.object_mask_threshold = 0.05
    net.log = lambda *x, **k: None
    batch = train_batch(make_scene, M, 0)

    def one():
        torch.manual_seed(0)
        net.zero_grad(set_to_none=True)
        net.step(batch, "train")["loss"].backward()

    times = {False: [], True: []}
    for i in range(a.warmup + a.steps):
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            t = timed(one)
            if i >= a.warmup:
                times[on].append(t)
    out = {"train_step": f"Net.step(batch, 'train') + backward, M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": gpu_state()}
    for on in (False, True):
        set_hooks(hooks, on)
        crit, shapes = criterion_time(net, one, 3)
        top, ours, cost = kernel_table(one)
        fig = dict(stats(times[on]), **crit, **counted(one), top_kernels=top)
        if on:
            fig["setloss_kernels"] = ours
            need = sum(4 * n * q + 4 * n * ((t + 31) // 32) for n, q, t in shapes)
            fig["levels_N_Q_T"] = shapes
            fig["match_cost_bytes"] = need
            fig["match_cost_bytes_at_3.35TBps_ms"] = round(need / HBM_BYTES_PER_S * 1e3, 4)
            if cost is not None:
                fig["match_cost_kernel_calls_ms"] = [cost[0], round(cost[1], 3)]
        out["criterion_on" if on else "criterion_off"] = fig
    hooks.uninstall()
    del net, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="+", default=[1, 2])
    ap.add_argument("--steps", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("criterion_hook_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("criterion_hook_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    for M in a.subnets:
        print(json.dumps(run(M, a, hooks, make_scene)), flush=True)


if __name__ == "__main__":
    main()
