"""Scene preparation cost: scenes.prepare on the device against the reference's KittiDataset.__getitem__ on the CPU.

    python tools/scene_prep_bench.py [--reps 20] [--warmup 3] [--seed 0] [--out result.json]

Writes a full-size synthetic SemanticKITTI tree to a temporary directory (seed-generated: 256 x 256 x 32 label volumes
with 19 classes and 30 instances, about 120k points per scan with the 283 input features) and reports, in one run:
  * device time per batch of scenes.prepare (CUDA events around the call, after warm-up; median, min and max) for
    train at M = 1 and M = 2 (rotation, flip, translation, crop) and val at M = 2 (TTA poses);
  * the host's file reading and draws per batch (SemanticKittiScenes.__getitem__), separately;
  * when build() staged the reference under oracle/_ref, the reference's __getitem__ on the same tree and the same
    draws on this machine's CPU, with one thread (as a DataLoader worker runs) and with all threads;
  * the GPU's name and power limit, which belong beside the device times.
"""
import argparse
import json
import os
import pickle
import random
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

from pasco_b200 import scenes as SC  # noqa: E402

SHAPE = (256, 256, 32)
N_POINTS, N_TTA, V, E = 120_000, 2, 19, 256
SCANS = [("00", "000000"), ("00", "000005"), ("01", "000000"), ("08", "000000")]
CONFIGS = {"train_m1": dict(split="train", n_subnets=1), "train_m2": dict(split="train", n_subnets=2),
           "val_m2": dict(split="val", n_subnets=2)}
AUG = dict(data_aug=True, max_angle=30.0, translate_distance=0.2, scale_range=0.05)


def scene(g):
    """19 classes (ground, structures, vegetation, poles, 8 thing classes) and 30 instances of thing classes."""
    sem = np.zeros(SHAPE, np.uint8)
    inst = np.zeros(SHAPE, np.uint8)
    sem[:, :, :3] = 255
    sem[:, :, 3:5] = 9
    sem[:, 100:130, 3:6] = 10
    sem[:, 130:150, 3:6] = 11
    sem[:, 150:175, 3:6] = 12
    sem[:, 175:, 3:5] = 17
    for cls in (13, 14, 15, 16, 18, 19):
        for _ in range(6):
            sx, sy, sz = g.integers(1, 30, 3)
            x, y = g.integers(0, 256 - sx), g.integers(0, 256 - sy)
            sem[x:x + sx, y:y + sy, 5:5 + min(sz, 20)] = cls
    x0, y0 = g.integers(150, 220, 2)
    sem[x0:x0 + 30, y0 - 40:y0, 5:20] = 255
    for i in range(30):
        cls = 1 + i % 8
        sx, sy, sz = g.integers(3, 20), g.integers(3, 10), g.integers(4, 12)
        x, y = g.integers(0, 256 - sx), g.integers(0, 256 - sy)
        sem[x:x + sx, y:y + sy, 5:5 + sz] = cls
        inst[x:x + sx, y:y + sy, 5:5 + sz] = i + 1
    return sem, inst


def write_tree(root, seed):
    g = np.random.default_rng(seed)

    def put(rel, data):
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data)
    for seq in range(11):
        s = f"{seq:02d}"
        eye = " ".join(f"{v:.1f}" for v in np.eye(4)[:3].ravel())
        put(f"dataset/sequences/{s}/calib.txt", f"P0: {eye}\nTr: {eye}\n".encode())
        put(f"dataset/sequences/{s}/times.txt", b"0.0\n" * 12)
        put(f"dataset/sequences/{s}/poses.txt", f"{eye}\n".encode() * 12)     # a pose per frame up to 000011
    for seq, frame in SCANS:
        put(f"dataset/sequences/{seq}/voxels/{frame}.bin", b"")
        sem, inst = scene(g)
        put(f"preprocess/instance_labels_v2/{seq}/{frame}_1_1.pkl",
            pickle.dumps({"semantic_labels": sem, "instance_labels": inst}))
        lo, hi = np.array([-2.0, -27.0, -3.0]), np.array([53.0, 27.0, 5.0])
        xyz = (lo + (hi - lo) * g.random((N_POINTS, 3))).astype(np.float32)
        coords = np.concatenate([xyz, g.random((N_POINTS, 1), dtype=np.float32)], 1)
        feats = {"coords": coords, "vote": g.standard_normal((N_POINTS, V), dtype=np.float32),
                 "embedding": g.standard_normal((N_TTA, E, N_POINTS), dtype=np.float32).astype(np.float16)}
        put(f"preprocess/waffleiron_v2/sequences/{seq}/seg_feats_tta/{frame}.pkl", pickle.dumps(feats))
        put(f"dataset/sequences/{seq}/labels/{frame}.label", g.integers(0, 1 << 20, N_POINTS, dtype=np.int32).tobytes())
    put("semantic-kitti.yaml", b"learning_map:\n  0: 0\n  10: 1\n")


def spread(xs):
    return {"median": statistics.median(xs), "min": min(xs), "max": max(xs), "n": len(xs)}


def device_times(root, cfg, reps, warmup, seed):
    ds = SC.SemanticKittiScenes(root=root, preprocess_root=os.path.join(root, "preprocess"), **cfg, **AUG)
    host, dev = [], []
    for r in range(warmup + reps):
        np.random.seed(seed + r)
        random.seed(seed + r)
        t0 = time.perf_counter()
        raw = ds[r % len(ds)]
        t1 = time.perf_counter()
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        start.record()
        SC.prepare(raw, "cuda")
        end.record()
        end.synchronize()
        if r >= warmup:
            host.append((t1 - t0) * 1e3)
            dev.append(start.elapsed_time(end))
    return {"device_ms": spread(dev), "host_read_ms": spread(host)}


def reference_times(root, cfg, reps, seed, threads):
    ref = os.path.join(ROOT, "oracle", "_ref")
    sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), ref]
    import pasco.data.semantic_kitti.kitti_dataset as KD
    torch.set_num_threads(threads)
    ds = KD.KittiDataset(root=root, preprocess_root=os.path.join(root, "preprocess"),
                         config_path=os.path.join(root, "semantic-kitti.yaml"), **cfg, **AUG)
    ts = []
    for r in range(reps):
        np.random.seed(seed + r)
        random.seed(seed + r)
        t0 = time.perf_counter()
        ds[r % len(ds)]
        ts.append((time.perf_counter() - t0) * 1e3)
    return spread(ts)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--ref-reps", type=int, default=2)
    ap.add_argument("--seed", type=int, default=0)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("scene_prep_bench: needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                       text=True)
    res = {"gpu": q.stdout.strip().splitlines()[0] if q.returncode == 0 else torch.cuda.get_device_name(),
           "cpu_threads": os.cpu_count(), "points_per_scan": N_POINTS}
    with tempfile.TemporaryDirectory() as root:
        write_tree(root, a.seed)
        for name, cfg in CONFIGS.items():
            res[name] = device_times(root, cfg, a.reps, a.warmup, a.seed)
        if os.path.isdir(os.path.join(ROOT, "oracle", "_ref", "pasco")):
            for name, cfg in CONFIGS.items():
                res[name]["reference_cpu_ms"] = {
                    "1_thread": reference_times(root, cfg, a.ref_reps, a.seed, 1),
                    "all_threads": reference_times(root, cfg, a.ref_reps, a.seed, os.cpu_count() or 1)}
    line = json.dumps(res)
    print(line)
    if a.out:
        with open(a.out, "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
