"""Inference time of PascoNet: the eval-mode forward without gradients (scripts/eval.py's network call: model.eval(),
forward(test=True)) on the benchmark scene, with launches per scene and peak memory.

    python tools/infer_bench.py [--subnets 1 3] [--scenes 20] [--warmup 3] [--root TREE] [--profile DIR]

Workload: configs[1] scale, 256x256x32 @10 % scenes (four seeds, device-resident before timing), f = 64, M = 1 and M = 3
subnets.  The network has recipe-free random weights; its BatchNorm running statistics are calibrated first (momentum None,
one train-mode forward under no_grad on a scene of another seed) so that eval mode sees realistic activations — after
~40 layers the default statistics (mean 0, variance 1) would keep almost no voxels.  Each scene is timed with CUDA
events around the forward and ended by a device synchronise; the median over --scenes scenes is reported after --warmup
scenes.  One more scene with ops.PROFILE gives the convolution launches per path, and the C-ABI call count
(ops.CALLS; each call launches one or more kernels of ours) gives the launches per scene.  The card's name, power limit
and SM clock are read right after the timed scenes.  --profile DIR writes per-kernel totals of one more scene under
torch.profiler (a separate run of the forward: tracing slows the host) to DIR/infer_kernels_M<M>_<tag>.json.

--root imports pasco_b200 from another source tree with its library built (a checkout of an earlier commit), so that two
builds can be alternated in one session; the tool uses only interfaces that earlier builds have.  Prints one JSON line
per subnet count; writes only under --profile.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

GRID, OCC, IN_CH, N_CLASSES = (256, 256, 32), 0.10, 283, 20


def gpu_state():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm",
                            "--format=csv,noheader,nounits", "-i", str(torch.cuda.current_device())],
                           capture_output=True, text=True, timeout=10)
        name, watts, sm, sm_max = [x.strip() for x in r.stdout.strip().split(",")]
        return {"name": name, "power_limit_w": float(watts), "sm_mhz": int(float(sm)), "sm_max_mhz": int(float(sm_max))}
    except Exception:
        return {"name": torch.cuda.get_device_name()}


def scene_on_device(make_scene, M, seed):
    sc = make_scene(GRID, OCC, M, IN_CH, N_CLASSES, seed=seed)
    d = lambda t: t.to("cuda")  # noqa: E731
    return dict(sc, in_feats=[d(t) for t in sc["in_feats"]], in_coords=[d(t) for t in sc["in_coords"]])


def calibrated_net(PascoNet, make_scene, M):
    torch.manual_seed(0)
    net = PascoNet(n_classes=N_CLASSES, n_infers=M, in_channels=IN_CH, f=64, num_queries=100).cuda()
    for m in net.modules():
        if isinstance(m, torch.nn.modules.batchnorm._BatchNorm):
            m.momentum = None
            m.num_batches_tracked.zero_()
    net.train()
    with torch.no_grad():
        forward(net, scene_on_device(make_scene, M, 100))
    return net.eval()


def forward(net, sc):
    return net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"],
               test=True)


def run(M, a, ops, PascoNet, make_scene):
    net = calibrated_net(PascoNet, make_scene, M)
    scenes = [scene_on_device(make_scene, M, seed) for seed in range(4)]
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    times, calls, voxels = [], [], []
    with torch.no_grad():
        for i in range(a.warmup + a.scenes):
            sc = scenes[i % len(scenes)]
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            c0 = ops.CALLS
            e0.record()
            out = forward(net, sc)
            e1.record()
            torch.cuda.synchronize()
            if i >= a.warmup:
                times.append(e0.elapsed_time(e1))
                calls.append(ops.CALLS - c0)
                voxels.append(int(out["sem_logits_at_scales"][1][0].F.shape[0]))
            del out
        gpu = gpu_state()
        ops.PROFILE = []
        forward(net, scenes[0])
        torch.cuda.synchronize()
        prof, ops.PROFILE = ops.PROFILE, None
        ops.PAIR_COUNTS.clear()
        census = {}
        for kind, e0, e1, m in prof:
            c = census.setdefault(f"{kind}/{m['path']}", {"launches": 0, "ms": 0.0})
            c["launches"] += 1
            c["ms"] += e0.elapsed_time(e1)
        for c in census.values():
            c["ms"] = round(c["ms"], 2)
        kernels = None
        if a.profile:
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                forward(net, scenes[0])
                torch.cuda.synchronize()
            kernels = {}
            for ev in p.events():
                if ev.device_type == torch.autograd.DeviceType.CUDA:
                    k = kernels.setdefault(ev.name, {"count": 0, "us": 0.0})
                    k["count"] += 1
                    k["us"] += ev.device_time
            os.makedirs(a.profile, exist_ok=True)
            path = os.path.join(a.profile, f"infer_kernels_M{M}_{a.tag or 'run'}.json")
            top = dict(sorted(kernels.items(), key=lambda kv: -kv[1]["us"]))
            json.dump({"M": M, "tag": a.tag, "kernels": top}, open(path, "w"), indent=0)
    del net, scenes
    torch.cuda.empty_cache()
    srt = sorted(times)
    return {"M": M, "ms_per_scene_median": round(statistics.median(times), 2), "ms_per_scene_min": round(srt[0], 2),
            "ms_per_scene_max": round(srt[-1], 2), "scenes": a.scenes, "launch_calls_per_scene": statistics.median(calls),
            "conv_census": dict(sorted(census.items())), "scale1_voxels": voxels[0],
            "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 2),
            "profiler_kernel_launches": sum(k["count"] for k in kernels.values()) if kernels else None, "gpu": gpu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--subnets", type=int, nargs="+", default=[1, 3])
    ap.add_argument("--scenes", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="source tree to import pasco_b200 from (its library built)")
    ap.add_argument("--tag", default="", help="label copied into every result line")
    ap.add_argument("--profile", default=None, help="directory for the torch.profiler per-kernel totals")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("infer_bench.py: no CUDA device")
    sys.path.insert(0, os.path.abspath(a.root))
    from pasco_b200 import _lib, ops
    _lib.load()
    from pasco_b200.net3d import PascoNet
    from pasco_b200.synthetic import make_scene
    ops.set_precision(a.precision)
    for M in a.subnets:
        r = run(M, a, ops, PascoNet, make_scene)
        r.update(tag=a.tag, precision=a.precision, root=os.path.basename(os.path.abspath(a.root)))
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
