"""Training-step time of PascoNet at several network widths f (levels f, 2f, 4f, 4f) on the benchmark scene, with the
census of convolution launches per kernel path.

    python tools/width_bench.py [--widths 32 64 96 128] [--steps 6] [--warmup 3] [--root TREE]

One step = forward + loss + backward + fused AdamW on one 256x256x32 @10 % scene (bench.py's workload, which is fixed at
f = 64).  The step time is the median over --steps steps, each timed with CUDA events around the whole step and ended by
a device synchronise.  One extra step with ops.PROFILE recording gives the launch census: the number of forward,
input-gradient and weight-gradient launches per path (planes / regs / splitk / simt) and their summed event time.  The
card's name, power limit and SM clock are read right after each width's timed steps.  --root imports pasco_b200 from
another source tree with its library already built (e.g. a checkout of an earlier commit), so that two builds can be
alternated in one session.  Prints one JSON line per width and writes nothing.
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


def run_width(f, a, ops, PascoNet, total_loss, scenes):
    torch.manual_seed(0)
    net = PascoNet(n_classes=N_CLASSES, n_infers=1, in_channels=IN_CH, f=f, num_queries=100).cuda().train()
    params = [p for p in net.parameters() if p.requires_grad]
    opt = torch.optim.AdamW(params, lr=1e-4, weight_decay=1e-4, fused=True)

    def step(i):
        sc = scenes[i % len(scenes)]
        out = net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
        loss = total_loss(out, sc, N_CLASSES, net.class_frequencies)
        opt.zero_grad(set_to_none=True)
        loss.backward()
        torch.nn.utils.clip_grad_norm_(params, 0.5)
        opt.step()

    for i in range(a.warmup):
        step(i)
    torch.cuda.synchronize()
    times = []
    for i in range(a.steps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        step(i)
        e1.record()
        torch.cuda.synchronize()
        times.append(e0.elapsed_time(e1))
    gpu = gpu_state()
    ops.PROFILE = []
    step(a.steps)
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
    del net, opt, params
    torch.cuda.empty_cache()
    return {"f": f, "ms_per_step_median": round(statistics.median(times), 2), "ms_per_step_min": round(min(times), 2),
            "steps": a.steps, "simt_launches": sum(c["launches"] for k, c in census.items() if k.endswith("/simt")),
            "census": dict(sorted(census.items())), "peak_mem_gib": round(torch.cuda.max_memory_allocated() / 2**30, 1),
            "gpu": gpu}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--widths", type=int, nargs="+", default=[32, 64, 96, 128])
    ap.add_argument("--steps", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--precision", default="fp32", choices=["fp32", "bf16"])
    ap.add_argument("--root", default=os.path.dirname(os.path.dirname(os.path.abspath(__file__))),
                    help="source tree to import pasco_b200 from (its library built)")
    ap.add_argument("--tag", default="", help="label copied into every result line")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("width_bench.py: no CUDA device")
    sys.path.insert(0, os.path.abspath(a.root))
    from pasco_b200 import _lib, ops
    _lib.load()
    from pasco_b200.net3d import PascoNet
    from pasco_b200.losses import total_loss
    from pasco_b200.synthetic import make_scene
    ops.set_precision(a.precision)
    dev = torch.device("cuda")
    scenes = []
    for seed in (0, 1):
        sc = make_scene(GRID, OCC, 1, IN_CH, N_CLASSES, seed=seed)
        d = lambda t: t.to(dev)  # noqa: E731
        scenes.append(dict(sc, in_feats=[d(t) for t in sc["in_feats"]], in_coords=[d(t) for t in sc["in_coords"]],
                           sem_labels={k: d(v) for k, v in sc["sem_labels"].items()}, mask_classes=d(sc["mask_classes"])))
    for f in a.widths:
        torch.cuda.reset_peak_memory_stats()
        r = run_width(f, a, ops, PascoNet, total_loss, scenes)
        r.update(tag=a.tag, precision=a.precision)
        print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
