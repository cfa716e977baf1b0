"""The UNMODIFIED reference's Net.step(batch, "train") plus backward and Net.step_inference(batch, "test") on the drop-in,
with the trunk hook off and on (pasco_b200/hooks.py install(trunk=True)); the attention, post-processing, evaluation and
criterion hooks are on in both arms.

    python tools/trunk_hook_bench.py [--train 1 2] [--test 1 3] [--steps 6] [--warmup 1]

Workload: tools/criterion_hook_bench.py's training batch and tools/evaluate_hook_bench.py's test batch at 256x256x32
@10 % (f = 64, Q = 100), trunk off and on alternated step by step.  Per arm:
  * the step's median and range in ms (host clock, ended by a device synchronise);
  * the time inside each hooked function (CylinderFeat.forward, Augmenter.merge, UNet3DV2.dense_bottleneck), every
    call bracketed by device synchronises, in a separate pass (their backward runs inside loss.backward() and is not
    separated);
  * host synchronisations (torch.cuda.set_sync_debug_mode), kernel launches (torch.profiler) and peak memory.
Prints one JSON line per workload, with the card's name, power limit and SM clock read in the same run; writes nothing.
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
from evaluate_hook_bench import counted, fresh_metrics, stats, timed, with_gt  # noqa: E402
from infer_bench import GRID  # noqa: E402
from postprocess_bench import batch_of, calibrate, reference_net  # noqa: E402

HOOKED = (("pasco.models.unet3d_sparse_v2", "CylinderFeat", "forward"),
          ("pasco.models.augmenter", "Augmenter", "merge"),
          ("pasco.models.unet3d_sparse_v2", "UNet3DV2", "dense_bottleneck"))


def gpu_state():
    import subprocess
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip() or q.stderr.strip()


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=on)


def hooked_time(one, steps):
    """ms per step inside each hooked function, every call bracketed by device synchronises."""
    import importlib
    spent, saved = {}, []
    for mod, cls, name in HOOKED:
        c = getattr(importlib.import_module(mod), cls)
        fn = getattr(c, name)
        saved.append((c, name, fn))

        def wrap(fn=fn, key=f"{cls}.{name}"):
            def inner(*a, **k):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                out = fn(*a, **k)
                torch.cuda.synchronize()
                spent[key] = spent.get(key, 0.0) + (time.perf_counter() - t0) * 1e3
                return out
            return inner
        setattr(c, name, wrap())
    try:
        per = {}
        for _ in range(steps):
            spent.clear()
            one()
            for k, v in spent.items():
                per.setdefault(k, []).append(v)
    finally:
        for c, name, fn in saved:
            setattr(c, name, fn)
    return {k + "_ms": round(statistics.median(v), 2) for k, v in per.items()}


def alternate(one, hooks, a):
    times = {False: [], True: []}
    for i in range(a.warmup + a.steps):
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            t = timed(one)
            if i >= a.warmup:
                times[on].append(t)
    out = {}
    for on in (False, True):
        set_hooks(hooks, on)
        out["trunk_on" if on else "trunk_off"] = dict(stats(times[on]), **hooked_time(one, 3), **counted(one))
    hooks.uninstall()
    return out


def train(M, a, hooks, make_scene):
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

    out = {"workload": f"Net.step(batch, 'train') + backward, M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": gpu_state(), **alternate(one, hooks, a)}
    del net, batch
    torch.cuda.empty_cache()
    return out


def test(M, a, hooks, make_scene):
    net = reference_net(M)
    batch = with_gt(make_scene, batch_of(make_scene, M, 1), M, 1)
    set_hooks(hooks, False)
    calibrate(net, batch)
    net.object_mask_threshold = 0.05
    net.log = lambda *x, **k: None

    def one():
        fresh_metrics(net)
        torch.manual_seed(0)
        with torch.no_grad():
            net.step_inference(batch, "test", eval=True)

    out = {"workload": f"Net.step_inference(batch, 'test'), M = {M}, {'x'.join(map(str, GRID))} @10 %",
           "steps": a.steps, "gpu": gpu_state(), **alternate(one, hooks, a)}
    del net, batch
    torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--train", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--test", type=int, nargs="*", default=[1, 3])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("trunk_hook_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("trunk_hook_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    for M in a.train:
        print(json.dumps(train(M, a, hooks, make_scene)), flush=True)
    for M in a.test:
        print(json.dumps(test(M, a, hooks, make_scene)), flush=True)


if __name__ == "__main__":
    main()
