"""Net.evaluate_all of the UNMODIFIED reference on the drop-in, with the evaluation hook off and on
(pasco_b200/hooks.py install(evaluate=True)); the attention and post-processing hooks are on in both modes.

    python tools/evaluate_hook_bench.py [--subnets 1 3] [--scenes 6] [--warmup 1] [--train-steps 8]

Workload: tools/postprocess_bench.py's 256x256x32 @10 % scenes (f = 64, Q = 100, calibrated random weights,
object_mask_threshold 0.05) with a ground truth from the scene generator: the scale-1 semantic labels with an unknown
slab (x in [120, 130)) and its ten box masks.  Hooks off and on alternate scene by scene.  Per mode:
  (a) one evaluate_all call in test mode (compute_uncertainty=True) on the inputs step_inference hands it, per entry
      (M + 1 entries per scene), each call on fresh metric objects and ended by a device synchronise;
  (b) Net.step_inference(batch, "test", eval=True) per scene;
  (c) Net.step(batch, "train") plus backward at M = 1 and M = 2 at 256x256x32 @10 % on tools/dropin_scale_bench.py's
      training batch (evaluate_all runs on subnets 0 and M - 1 without uncertainty), hooks off and on alternated step
      by step over --train-steps steps after --warmup.
Each: median and range in ms, host synchronisations (torch.cuda.set_sync_debug_mode), kernel launches (torch.profiler,
CUDA activities) and peak memory of a separate pass.  (b) and (c) also give the time spent inside evaluate_all, from
separate passes in which every evaluate_all call is bracketed by device synchronises, and the number of calls the hook
sent to the saved original.  The bytes the dense passes must move are computed from the shapes.
Prints one JSON line per figure; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle", "_ref"), os.path.join(ROOT, "compat"),
                os.path.join(ROOT, "tests", "golden")]
from infer_bench import GRID, N_CLASSES, gpu_state  # noqa: E402
from postprocess_bench import batch_of, calibrate, reference_net  # noqa: E402


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=on)


def with_gt(make_scene, batch, M, seed):
    sc = make_scene(GRID, 0.10, M, 283, N_CLASSES, seed=seed)
    sem = sc["sem_labels"]["1_1"][0].clone()
    sem[120:130] = 255
    masks = torch.zeros((len(sc["mask_boxes"]),) + GRID, dtype=torch.bool)
    for i, (lo, hi) in enumerate(sc["mask_boxes"]):
        masks[i, lo[0]:hi[0], lo[1]:hi[1], lo[2]:hi[2]] = True
    ml = {"labels": sc["mask_classes"].cuda(), "masks": masks.cuda()}
    return dict(batch, semantic_label=sem[None].cuda(), semantic_label_origin=sem[None].cuda(), mask_label=[ml],
                mask_label_origin=[ml])


def stats(v):
    return {"ms_median": round(statistics.median(v), 2), "ms_min_max": [round(min(v), 2), round(max(v), 2)]}


def counted(fn):
    """(host synchronisations, kernel launches, peak GiB) of one call of fn."""
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    n_sync = sum("synchroniz" in str(x.message) for x in w)
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        fn()
        torch.cuda.synchronize()
    n_launch = sum(1 for ev in p.events() if ev.device_type == torch.autograd.DeviceType.CUDA)
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    fn()
    torch.cuda.synchronize()
    return {"host_syncs": n_sync, "kernel_launches": n_launch,
            "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2)}


def timed(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def fresh_metrics(net):
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics
    for i in net.pq_stat["test"]:
        net.pq_stat["test"][i] = PQStat()
        net.ssc_metrics["test"][i] = SSCMetrics(net.n_classes)
        net.uncertainty_metrics_by_thresholds[0.5][i] = UncertaintyMetrics()


def recorded_calls(net, batch):
    """The keyword arguments of every evaluate_all call of one step_inference(eval=True)."""
    cls = type(net)
    calls, inner = [], cls.evaluate_all

    def rec(self, **kw):
        calls.append(kw)
        return inner(self, **kw)
    cls.evaluate_all = rec
    try:
        with torch.no_grad():
            net.step_inference(batch, "test", eval=True)
    finally:
        cls.evaluate_all = inner
    return calls


def dense_bytes(K, cells, n_masks):
    """Bytes one hooked call (one entry) must move through its dense passes: the ground truth's uint8 mask stack and
    label read, its gt ids written (k_eval_gt), gt ids read and the fp32 gt volume written (k_eval_gt_volume), class
    planes + confidence + label read and the int64 argmax written (ssc_planes), ids + label + gt ids (pairs), ids +
    confidence + gt ids (vox)."""
    gt = cells * (n_masks + 1 + 4) + cells * (4 + 4)
    return gt + cells * (4 * K + 4 + 1 + 8) + cells * (4 + 1 + 4) + cells * (4 + 4 + 4)


def run(M, a, hooks, make_scene):
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics
    from pasco.loss.panoptic_quality import PQStat
    net = reference_net(M)
    set_hooks(hooks, False)
    net = calibrate(net, batch_of(make_scene, M, 100))
    net.object_mask_threshold = 0.05
    batches = [with_gt(make_scene, batch_of(make_scene, M, s), M, s) for s in range(2)]
    per_call = {False: [], True: []}
    step = {False: [], True: []}
    for i in range(a.warmup + a.scenes):
        b = batches[i % len(batches)]
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            fresh_metrics(net)
            with torch.no_grad():
                t = timed(lambda: net.step_inference(b, "test", eval=True))
            calls = recorded_calls(net, b)
            ts = []
            for kw in calls:
                kw = dict(kw, pq_stat=PQStat(), ssc_metrics=SSCMetrics(N_CLASSES), uncertainty_metrics=UncertaintyMetrics())
                ts.append(timed(lambda: net.evaluate_all(**kw)))
            if i >= a.warmup:
                step[on].append(t)
                per_call[on].extend(ts)
    out = {"M": M, "entries": M + 1, "scenes": a.scenes, "gpu": gpu_state()}
    K, cells = N_CLASSES, GRID[0] * GRID[1] * GRID[2]
    n_masks = batches[0]["mask_label_origin"][0]["masks"].shape[0]
    out["dense_pass_bytes_per_call"] = dense_bytes(K, cells, n_masks)
    out["dense_pass_floor_ms_at_3.35TBps"] = round(dense_bytes(K, cells, n_masks) / 3.35e12 * 1e3, 3)
    for on in (False, True):
        set_hooks(hooks, on)
        kw = recorded_calls(net, batches[0])[-1]

        def one_call():
            net.evaluate_all(**dict(kw, pq_stat=PQStat(), ssc_metrics=SSCMetrics(N_CLASSES),
                                    uncertainty_metrics=UncertaintyMetrics()))

        def one_step():
            fresh_metrics(net)
            with torch.no_grad():
                net.step_inference(batches[0], "test", eval=True)
        out["hooks_on" if on else "hooks_off"] = {
            "evaluate_all": dict(stats(per_call[on]), **counted(one_call)),
            "step_inference_eval": dict(stats(step[on]), **instrumented(net, one_step, 1), **counted(one_step))}
    hooks.uninstall()
    del net, batches
    torch.cuda.empty_cache()
    return out


def instrumented(net, fn, steps):
    """The median over `steps` calls of fn() of the ms spent inside evaluate_all (each of its calls bracketed by
    device synchronises, so these calls are not the timed ones) and the number of evaluate_all calls the hook sent to
    the saved original."""
    cls = type(net)
    inner, per_step, fallbacks = cls.evaluate_all, [], []
    orig = getattr(cls, "_pasco_b200_orig_evaluate_all", None)

    def timed_eval(self, **kw):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        r = inner(self, **kw)
        torch.cuda.synchronize()
        per_step[-1] += (time.perf_counter() - t0) * 1e3
        return r
    cls.evaluate_all = timed_eval
    if orig is not None and inner is not orig:                   # the hook is installed: spy on its fallbacks
        cls._pasco_b200_orig_evaluate_all = lambda *a, **k: fallbacks.append(1) or orig(*a, **k)
    try:
        for _ in range(steps):
            per_step.append(0.0)
            fn()
    finally:
        cls.evaluate_all = inner
        if orig is not None:
            cls._pasco_b200_orig_evaluate_all = orig
    return {"evaluate_all_ms_per_step_median": round(statistics.median(per_step), 1), "fallbacks": len(fallbacks)}


def train_figure(M, a, hooks, make_scene):
    """(c) at full scene size: tools/dropin_scale_bench.py's training batch (its scene, dense semantic labels and box
    masks, full-scene subnet frames) and Net, step + backward, hooks off / on alternated step by step."""
    from dropin_scale_bench import train_batch
    net = reference_net(M).train()
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1, device="cuda") for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K, device="cuda")
    net.object_mask_threshold = 0.05
    batch = train_batch(make_scene, M, 0)

    def one():
        torch.manual_seed(0)
        net.zero_grad(set_to_none=True)
        net.step(batch, "train")["loss"].backward()

    times = {False: [], True: []}
    for i in range(a.warmup + a.train_steps):
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            t = timed(one)
            if i >= a.warmup:
                times[on].append(t)
    out = {"train_step": f"Net.step(batch, 'train') + backward, M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.train_steps, "gpu": gpu_state()}
    for on in (False, True):
        set_hooks(hooks, on)
        out["hooks_on" if on else "hooks_off"] = dict(stats(times[on]), **instrumented(net, one, 3), **counted(one))
    hooks.uninstall()
    del net, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--scenes", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=1)
    ap.add_argument("--train-steps", type=int, default=8, help="0: no training-step figures")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("evaluate_hook_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("evaluate_hook_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    import pasco.models.metrics as MET
    from make_golden_eval import binary_calibration_error
    MET.binary_calibration_error = binary_calibration_error      # torchmetrics 1.4, as the reference computes it
    for M in a.subnets:
        print(json.dumps(run(M, a, hooks, make_scene)), flush=True)
    if a.train_steps:
        for M in (1, 2):
            print(json.dumps(train_figure(M, a, hooks, make_scene)), flush=True)


if __name__ == "__main__":
    main()
