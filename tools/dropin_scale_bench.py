"""The unmodified reference on the drop-in at full scene size (256x256x32 @10 %): does each run fit on the card, its peak
memory and its median time, with the attention hook (hooks.install: TransformerPredictorV2.forward on the device-built
mask bits) off and on.

    python tools/dropin_scale_bench.py [--eval-subnets 1 3] [--train-subnets 1 2] [--steps 3] [--warmup 1]

Runs, one JSON line each:
  eval   Net.step_inference(batch, "test") — scripts/eval.py's call — at each --eval-subnets M, hooks off
         (install nothing: the reference's own code) and hooks on (install(attention=True, postprocess=True)).
  train  Net.step(batch, "train") + backward of its loss — scripts/train.py's step — at each --train-subnets M, hooks off
         and on, on a reference-format batch from synthetic.make_scene: dense `mask_label` (the scene's boxes),
         `semantic_label`, `geo_labels`, `sem_labels`.
The reference Net has seeded random weights (f = 64, Q = 100); eval runs calibrate its BatchNorm statistics first, as
tools/postprocess_bench.py does.  A run that raises torch.OutOfMemoryError is reported with "completes": false, the
allocation it failed on and the peak reached; times are medians over --steps calls after --warmup, each ended by a device
synchronise.  The card's name and power limit are read in the same process.  Writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle", "_ref"), os.path.join(ROOT, "compat")]
from infer_bench import GRID, IN_CH, N_CLASSES, OCC, gpu_state  # noqa: E402
from postprocess_bench import batch_of, calibrate, reference_net  # noqa: E402


def train_batch(make_scene, M, seed):
    """A reference-format training batch: the scene of batch_of plus dense labels and instance masks."""
    from pasco_b200.synthetic import training_batch
    tb = training_batch(make_scene(GRID, OCC, M, IN_CH, N_CLASSES, seed=seed))
    b = batch_of(make_scene, M, seed)
    b.update({k: tb[k] for k in ("sem_labels", "semantic_label", "geo_labels", "mask_label")})
    return b


def measured(fn, steps, warmup):
    """→ {"completes", "peak_gib", "ms_median"} of fn() called warmup + steps times."""
    torch.cuda.empty_cache()
    torch.cuda.reset_peak_memory_stats()
    times = []
    try:
        for i in range(warmup + steps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            if i >= warmup:
                times.append((time.perf_counter() - t0) * 1e3)
        out = {"completes": True, "ms_median": round(statistics.median(times), 1)}
    except torch.OutOfMemoryError as e:
        out = {"completes": False, "error": str(e).split("\n")[0][:160]}
    torch.cuda.synchronize()
    out["peak_gib"] = round(torch.cuda.max_memory_allocated() / 2**30, 2)
    return out


def set_hooks(hooks, on):
    hooks.uninstall()
    if on:
        assert hooks.install(attention=True, postprocess=True)


def eval_run(M, a, hooks, make_scene):
    net = reference_net(M)
    set_hooks(hooks, False)
    net = calibrate(net, batch_of(make_scene, M, 100))
    net.object_mask_threshold = 0.05
    batch = batch_of(make_scene, M, 0)
    out = {"run": "eval", "call": 'Net.step_inference(batch, "test")', "M": M}
    with torch.no_grad():
        for on in (False, True):
            set_hooks(hooks, on)
            out["hooks_on" if on else "hooks_off"] = measured(lambda: net.step_inference(batch, "test"), a.steps,
                                                              a.warmup)
    hooks.uninstall()
    return out


def train_run(M, a, hooks, make_scene):
    net = reference_net(M).train()
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1, device="cuda") for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K, device="cuda")
    net.object_mask_threshold = 0.05
    batch = train_batch(make_scene, M, 0)

    def step():
        net.zero_grad(set_to_none=True)
        net.step(batch, "train")["loss"].backward()

    out = {"run": "train", "call": 'Net.step(batch, "train") + backward', "M": M}
    for on in (False, True):
        set_hooks(hooks, on)
        torch.manual_seed(0)
        out["hooks_on" if on else "hooks_off"] = measured(step, a.steps, a.warmup)
    hooks.uninstall()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--eval-subnets", type=int, nargs="*", default=[1, 3])
    ap.add_argument("--train-subnets", type=int, nargs="*", default=[1, 2])
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=1)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("dropin_scale_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("dropin_scale_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    runs = [(eval_run, M) for M in a.eval_subnets] + [(train_run, M) for M in a.train_subnets]
    for fn, M in runs:
        res = fn(M, a, hooks, make_scene)
        print(json.dumps(dict(res, scene=f"{GRID[0]}x{GRID[1]}x{GRID[2]} @{OCC:.0%}", gpu=gpu_state())), flush=True)
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
