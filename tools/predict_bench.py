"""Time of PascoNet.predict on the benchmark scene: the eval forward and the post-processing (csrc/panoptic.cu through
predict.postprocess) timed separately, and the post-processing against the torch restatement of the same computation
(ensemble.py) on the same network outputs, alternated in one process.

    python tools/predict_bench.py [--subnets 1 3] [--scenes 20] [--warmup 3]

Workload: configs[1] scale, 256x256x32 @10 % scenes (four seeds, device-resident), f = 64, Q = 100, M = 1 and M = 3
subnets, the network calibrated as tools/infer_bench.py does (running statistics from one train-mode forward on a scene of
another seed), identity poses.  Per scene: CUDA events around the forward, then around the post-processing of its
outputs, then around the torch path on the same outputs, each ended by a device synchronise; medians over --scenes scenes
after --warmup.  The thresholds are the reference's except object_mask_threshold = 0.05 (a calibrated but untrained
network's class probabilities rarely reach 0.7, and the panoptic passes should see kept queries).  One more scene runs
under torch.profiler (a separate call: tracing slows the host) and gives the kernel launches of the post-processing and
the device time of panoptic passes 1 and 2 with the bytes each must move (pass 1: the [N, Q] probabilities read once +
12 B of record per row; pass 2: the 12 B records read + 12 B of outputs per row).  Host synchronisations come from
torch.cuda.set_sync_debug_mode.  Prints one JSON line per subnet count; writes nothing.
"""
import argparse
import json
import os
import statistics
import sys
import warnings

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

THR = dict(overlap_threshold=0.4, object_mask_threshold=0.05, iou_threshold=0.2)
HBM_BYTES_PER_S = 3.35e12           # NVIDIA H100 SXM data sheet


def timed(fn):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    out = fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), out


def outputs(ret):
    preds = [{"voxel_logits": (p["voxel_logits"].F, p["voxel_logits"].C), "query_logits": p["query_logits"]}
             for p in ret["panop_predictions"]]
    return preds, [(s.F, s.C) for s in ret["sem_logits_at_scales"][1]]


def torch_path(preds, sems, Ts):
    from pasco_b200 import ensemble as E
    p3 = [{"voxel_logits": (p["voxel_logits"][0], p["voxel_logits"][1][:, 1:]), "query_logits": p["query_logits"]}
          for p in preds]
    s3 = [(f, c[:, 1:]) for f, c in sems]
    sem_denses = E.ensemble_sem_compl(s3, Ts)
    out = E.ensemble_panop(p3, sem_denses, Ts, iou_threshold=THR["iou_threshold"])
    return [E.panoptic_inference_with_confidence(o["voxel_probs"][0], o["query_probs"][0], THR["overlap_threshold"],
                                                 THR["object_mask_threshold"], [1, 2, 3, 4, 5, 6, 7, 8]) for o in out]


def run(M, a):
    from infer_bench import calibrated_net, gpu_state, scene_on_device
    from pasco_b200 import ops, predict as P
    from pasco_b200.net3d import PascoNet
    from pasco_b200.synthetic import make_scene
    net = calibrated_net(PascoNet, make_scene, M)
    scenes = [scene_on_device(make_scene, M, seed) for seed in range(4)]
    Ts = [torch.eye(4) for _ in range(M)]
    t_fwd, t_post, t_torch = [], [], []
    with torch.no_grad():
        for i in range(a.warmup + a.scenes):
            sc = scenes[i % len(scenes)]
            tf, ret = timed(lambda: net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"],
                                        sc["min_Cs"], sc["max_Cs"], test=True))
            preds, sems = outputs(ret)
            tp, ent = timed(lambda: P.postprocess(preds, sems, Ts, **THR))
            tt, _ = timed(lambda: torch_path(preds, sems, Ts))
            if i >= a.warmup:
                t_fwd.append(tf)
                t_post.append(tp)
                t_torch.append(tt)
        gpu = gpu_state()
        # one more scene: host synchronisations, calls, peak memory, then the kernels under the profiler
        ret = net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"],
                  test=True)
        preds, sems = outputs(ret)
        torch.cuda.synchronize()
        stats = {}
        for name, fn in (("engine", lambda: P.postprocess(preds, sems, Ts, **THR)), ("torch", lambda: torch_path(preds, sems, Ts))):
            calls0 = ops.CALLS
            torch.cuda.reset_peak_memory_stats()
            base = torch.cuda.memory_allocated()
            with warnings.catch_warnings(record=True) as w:
                warnings.simplefilter("always")
                torch.cuda.set_sync_debug_mode("warn")
                try:
                    fn()
                finally:
                    torch.cuda.set_sync_debug_mode("default")
            stats[name] = {"cabi_calls": ops.CALLS - calls0,
                           "host_syncs": sum("synchroniz" in str(x.message) for x in w),
                           "peak_mb": round((torch.cuda.max_memory_allocated() - base) / 2 ** 20, 1)}
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            ent = P.postprocess(preds, sems, Ts, **THR)
            torch.cuda.synchronize()
    kernels = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "Memcpy" not in e.name
               and "Memset" not in e.name]
    passes = {}
    for key in ("k_panoptic_pass1", "k_panoptic_pass2"):
        ev = [e for e in kernels if key in e.name]
        passes[key] = (len(ev), sum(e.device_time for e in ev) / 1e3)          # launches, ms
    rows = sum(e["lin"].numel() for e in ent)
    cols = [(e["lin"].numel(), e["query_probs"].shape[0]) for e in ent]
    p1_bytes = sum(n * q * 4 + 12 * n for n, q in cols)
    p2_bytes = sum(24 * n for n, _ in cols)
    res = {"subnets": M, "queries": 100, "entries": len(ent), "rows_per_entry": [n for n, _ in cols],
           "queries_per_entry": [q for _, q in cols], "segments_per_entry": [len(e["segments_info"]) for e in ent],
           "forward_ms_median": round(statistics.median(t_fwd), 3),
           "postprocess_ms_median": round(statistics.median(t_post), 3),
           "torch_path_ms_median": round(statistics.median(t_torch), 3),
           "postprocess_share_of_predict": round(statistics.median(t_post) / (statistics.median(t_fwd) + statistics.median(t_post)), 4),
           "kernel_launches_postprocess": len(kernels), "rows_total": rows,
           **{f"{k}_{s}": v for k, d in stats.items() for s, v in d.items()}}
    for key, b in (("k_panoptic_pass1", p1_bytes), ("k_panoptic_pass2", p2_bytes)):
        n, ms = passes[key]
        res[f"{key}_launches"] = n
        res[f"{key}_ms"] = round(ms, 4)
        res[f"{key}_bytes"] = b
        res[f"{key}_hbm_frac"] = round(b / (ms * 1e-3) / HBM_BYTES_PER_S, 4) if ms > 0 else None
    res["gpu"] = gpu
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--scenes", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "predict_bench measures on the GPU"
    from pasco_b200 import ops
    ops.set_precision("fp32")
    for M in a.subnets:
        print(json.dumps(run(M, a)), flush=True)


if __name__ == "__main__":
    main()
