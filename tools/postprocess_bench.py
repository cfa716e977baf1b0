"""Test-time step of the UNMODIFIED reference on the drop-in, with the post-processing hooks off and on: scripts/eval.py's
Net.step_inference(batch, "test") → forward, Ensembler.ensemble_sem_compl / ensemble_panop and panoptic_inference per
entry (net_panoptic_sparse.py:539-648), eval=False (the metric objects are out of the hooks' scope).

    python tools/postprocess_bench.py [--subnets 1 3] [--occ 0.10] [--scenes 10] [--warmup 2] [--train-steps 6]

Workload: the 256x256x32 @10 % scenes of tools/infer_bench.py (four seeds, device-resident), f = 64, Q = 100, M = 1 and
M = 3, under the scene generator's poses.  The reference Net has recipe-free random weights; its BatchNorm running
statistics are calibrated as infer_bench.py calibrates PascoNet's (momentum None, one train-mode forward under no_grad on a
scene of another seed), with is_predict_panop=False: the reference's train-mode transformer builds a [800, P] attention
mask reduction of 37 GiB at this scale.  object_mask_threshold is lowered to 0.05 so that segments survive the untrained query heads.  The
attention hooks are on in both modes, so the forward is the same and the two modes differ only in the post-processing.
Each scene is timed around step_inference, ended by a device synchronise; hooks off and on alternate scene by scene.
Per mode: the median total, the reference's own inference_times (the forward, which it times with synchronises), the
remainder (ensembling + panoptic inference), the peak memory of separate passes, the host synchronisations of one scene
(torch.cuda.set_sync_debug_mode) and the kernel launches of one scene (torch.profiler, CUDA activities).  --occ lowers the
occupancy (at M = 3 the reference's own forward does not fit on an 80 GB card at 10 % or 5 %:
transformer_predictor_v2.py:164 sums the [800, P] attention mask in int64).

The training-step figure: Net.step(batch, "train") (scripts/train.py's step: forward, criterion, and panoptic_inference
plus evaluate_all on subnets 0 and M − 1) at M = 2 on the 64x64x8 @5 % scene of the eval fixtures with recipe weights and
a seeded ground truth (the reference's train-mode transformer does not fit at 256x256x32), hooks off and on alternated
over --train-steps steps, timed from the call to a device synchronise, no backward.  Prints one JSON line per subnet count
and one for the training step; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import time
import warnings

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle", "_ref"), os.path.join(ROOT, "compat")]
from infer_bench import GRID, IN_CH, N_CLASSES, OCC, gpu_state  # noqa: E402


def reference_net(M):
    import MinkowskiEngine as ME  # noqa: F401  (compat → pasco_b200.me)
    from pasco.models.net_panoptic_sparse import Net
    torch.manual_seed(0)
    freqs = {f"1_{s}": np.ones(N_CLASSES) for s in (1, 2, 4)}
    return Net(n_classes=N_CLASSES, class_names=[str(i) for i in range(N_CLASSES)], class_weights=torch.ones(N_CLASSES),
               encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3, dense3d_dropout=0.0, n_infers=M,
               class_frequencies=freqs, in_channels=IN_CH, num_queries=100, f=64).cuda()


def batch_of(make_scene, M, seed, occ=OCC):
    sc = make_scene(GRID, occ, M, IN_CH, N_CLASSES, seed=seed)
    d = lambda t: t.to("cuda")  # noqa: E731
    return dict(in_feats=[d(t) for t in sc["in_feats"]], in_coords=[d(t) for t in sc["in_coords"]],
                min_Cs=[d(t) for t in sc["min_Cs"]], max_Cs=[d(t) for t in sc["max_Cs"]], Ts=[d(t) for t in sc["Ts"]],
                global_min_Cs=d(sc["global_min_Cs"]), global_max_Cs=d(sc["global_max_Cs"]),
                geo_labels={k: d(v) for k, v in sc["sem_labels"].items()})


def calibrate(net, batch):
    for m in net.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = None
            m.num_batches_tracked.zero_()
    net.train()
    import MinkowskiEngine as ME
    with torch.no_grad():
        in_coords, in_feats = net.feat(batch["in_feats"], batch["in_coords"])
        x = net.augmenter.merge(ME.SparseTensor(in_feats, in_coords.int()))
        net(x, 1, batch["geo_labels"], global_min_coords=batch["global_min_Cs"], global_max_coords=batch["global_max_Cs"],
            min_Cs=batch["min_Cs"], max_Cs=batch["max_Cs"], Ts=batch["Ts"], is_predict_panop=False, return_ensemble=False)
    return net.eval()


def set_hooks(hooks, on):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=on)


def one(net, batch):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    net.step_inference(batch, "test", measure_time=True)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, net.inference_times[-1] * 1e3


def syncs(net, batch):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            net.step_inference(batch, "test")
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return sum("synchroniz" in str(x.message) for x in w)


def launches(net, batch):
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as p:
        net.step_inference(batch, "test")
        torch.cuda.synchronize()
    return sum(1 for ev in p.events() if ev.device_type == torch.autograd.DeviceType.CUDA)


def run(M, a, hooks, make_scene):
    net = reference_net(M)
    set_hooks(hooks, False)
    net = calibrate(net, batch_of(make_scene, M, 100, a.occ))
    net.object_mask_threshold = 0.05
    batches = [batch_of(make_scene, M, seed, a.occ) for seed in range(4)]
    res = {False: {"total": [], "fwd": []}, True: {"total": [], "fwd": []}}
    with torch.no_grad():
        for i in range(a.warmup + a.scenes):
            for on in (False, True) if i % 2 == 0 else (True, False):
                set_hooks(hooks, on)
                total, fwd = one(net, batches[i % len(batches)])
                if i >= a.warmup:
                    res[on]["total"].append(total)
                    res[on]["fwd"].append(fwd)
        gpu = gpu_state()
        out = {"M": M, "scenes": a.scenes, "gpu": gpu}
        for on in (False, True):
            set_hooks(hooks, on)
            torch.cuda.empty_cache()
            torch.cuda.reset_peak_memory_stats()
            one(net, batches[0])
            peak = torch.cuda.max_memory_allocated() / 2**30
            r = res[on]
            rem = [t - f for t, f in zip(r["total"], r["fwd"])]
            out["hooks_on" if on else "hooks_off"] = {
                "total_ms_median": round(statistics.median(r["total"]), 1),
                "forward_ms_median": round(statistics.median(r["fwd"]), 1),
                "postprocess_ms_median": round(statistics.median(rem), 1),
                "postprocess_ms_min_max": [round(min(rem), 1), round(max(rem), 1)],
                "peak_mem_gib": round(peak, 2), "host_syncs": syncs(net, batches[0]),
                "kernel_launches": launches(net, batches[0])}
    hooks.uninstall()
    del net, batches
    torch.cuda.empty_cache()
    return out


def train_figure(a, hooks):
    sys.path.insert(0, os.path.join(ROOT, "tests", "golden"))
    import parity
    from recipe import fill_state_dict
    _, net = parity.reference_net(n_infers=2)
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1) for _ in range(2)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    net.to(dev).train()
    meta = parity.INFER_MANIFEST["cases"]["m2"]
    sc = parity.scene(meta, 2)
    grid = tuple(meta["grid"])
    g = torch.Generator().manual_seed(5)
    sem = torch.randint(0, K, (2,) + grid, generator=g)
    sem[torch.rand(sem.shape, generator=g) < 0.6] = 0
    sem[:, :, :2, :] = 255
    masks = []
    for m in range(2):
        present = [c for c in range(1, K) if (sem[m] == c).any()]
        masks.append({"labels": torch.tensor(present, dtype=torch.uint8, device=dev),
                      "masks": torch.stack([sem[m] == c for c in present]).to(dev)})
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 sem_labels=sc["sem_labels"], semantic_label=sem.to(torch.uint8).to(dev),
                 geo_labels={"1_1": torch.where(sem == 255, 255.0, (sem > 0).float()).to(dev)}, mask_label=masks)
    times = {False: [], True: []}
    for i in range(2 + a.train_steps):
        for on in (False, True) if i % 2 == 0 else (True, False):
            set_hooks(hooks, on)
            torch.manual_seed(0)
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            net.step(batch, "train")
            torch.cuda.synchronize()
            if i >= 2:
                times[on].append((time.perf_counter() - t0) * 1e3)
    hooks.uninstall()
    return {"train_step": "Net.step(batch, 'train'), M = 2, 64x64x8 @5 %", "steps": a.train_steps,
            "hooks_off_ms_median": round(statistics.median(times[False]), 1),
            "hooks_on_ms_median": round(statistics.median(times[True]), 1), "gpu": gpu_state()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--scenes", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--occ", type=float, default=OCC)
    ap.add_argument("--train-steps", type=int, default=6, help="0: no training-step figure")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("postprocess_bench.py: no CUDA device")
    if not os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
        raise SystemExit("postprocess_bench.py: the reference is not staged under oracle/_ref (run build())")
    from pasco_b200 import _lib, hooks, ops
    _lib.load()
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    for M in a.subnets:
        print(json.dumps(dict(run(M, a, hooks, make_scene), occ=a.occ)), flush=True)
    if a.train_steps:
        print(json.dumps(train_figure(a, hooks)), flush=True)


if __name__ == "__main__":
    main()
