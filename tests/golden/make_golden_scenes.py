"""Golden vectors for pasco_b200/scenes.py — BUILD CONTAINER ONLY: writes a small synthetic SemanticKITTI tree to a
temporary directory and runs the reference's OWN, unmodified `KittiDataset.__getitem__`
(pasco/data/semantic_kitti/kitti_dataset.py:126-490, collate.py) on it on the CPU under fixed seeds.

    python tests/golden/make_golden_scenes.py

The tree: sequences 00-10 with calib.txt, times.txt and poses.txt; voxels/*.bin naming the scans (000003 is skipped by
frame_interval = 5); per scan the label pickle (256 x 256 x 32 semantic and instance volumes), the WaffleIron pickle
(coords [N, 4] fp32, vote [N, 19] fp32, embedding [2, 256, N] fp16 — the reference's 283 input features) and the
.label words (upper 16 bits set, dropped by the reader).  Scan 08/000005 has no instance.

Cases (np.random.seed / random.seed before __getitem__):
  train_rot   train, M = 2, 30° rotation, flip, translation, 5 % scale, crop
  val_tta     val, M = 2, data_aug (TTA poses), no crop
  no_inst     val, M = 1, no augmentation, the scan without instances
  identity    train, M = 2, max_angle = 0 and no scale: T is a flip and a translation whose offsets lie away from a
              rounding tie on every axis, so every coordinate is exact whatever the summation order

Stored (scenes_semkitti.npz, compressed): every file of the tree as bytes under "tree/<path>"; per case its arguments
and draws (item order, embedding indices, crop draws) and every field collate_fn returns, per item, in the smallest form
that keeps its values: in_feats as its computed columns plus each row's point index into the scan's WaffleIron arrays
(vote, intensity and embedding are copies of them); the scale-1 volumes as one uint8 array [5, X, Y, Z] of
semantic_label, instance_label, geo_labels["1_1"] and the mask stack's per-cell stuff and instance index + 1 (0 = none;
the stuff masks are disjoint, and so are the instance masks), the untransformed frame's mask indices likewise [2, ...]
once per scan under "origin/<seq>/<frame>";
in_coords as int16 and the point labels as uint16 (the reference's dtypes are stored beside them),
sem_labels["1_1"] once as semantic_label (the reference returns the same tensor), and the untransformed volumes not at
all: this script checks that they are the scans' label volumes, stacked.  Point coordinates are multiples of 1/64 m
and the copied features (vote, embedding) follow a pattern, so the file stays small.
"""
import json
import os
import pickle
import random
import sys
import tempfile

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import stage_reference  # noqa: E402

sys.path[:0] = [os.path.join(ROOT, "oracle", "shims"), os.path.join(ROOT, "compat"), stage_reference.source()]

import numpy as np  # noqa: E402
import torch  # noqa: E402

SHAPE = (256, 256, 32)
SCANS = {("00", "000000"): True, ("00", "000005"): True, ("00", "000010"): True, ("01", "000000"): True,
         ("08", "000000"): True, ("08", "000005"): False}          # → has instances
SKIPPED = [("00", "000003")]
N_POINTS, N_TTA, V, E = 1000, 2, 19, 256
THING_IDS = [1, 2, 3, 4, 5, 6, 7, 8]
OWN_COLUMNS = [V + 1] + list(range(V + 2 + E, V + 2 + E + 6))     # in_feats columns computed, not copied (4 coords)
CASES = {
    "train_rot": dict(split="train", n_subnets=2, data_aug=True, max_angle=30.0, translate_distance=0.2,
                      scale_range=0.05, idx=0, seed=1),
    "val_tta": dict(split="val", n_subnets=2, data_aug=True, max_angle=30.0, translate_distance=0.2, scale_range=0.0,
                    idx=0, seed=2),
    "no_inst": dict(split="val", n_subnets=1, data_aug=False, max_angle=30.0, translate_distance=0.2, scale_range=0.0,
                    idx=1, seed=3),
    "identity": dict(split="train", n_subnets=2, data_aug=True, max_angle=0.0, translate_distance=0.2,
                     scale_range=0.0, idx=2, seed=4),
}


def scene(seed, with_instances):
    """Label volumes: unknown (255) below the ground and in a far blob, road / sidewalk / terrain ground, buildings,
    vegetation and poles, and things (cars, persons, bicycles, trucks) with instance ids."""
    g = np.random.default_rng(seed)
    sem = np.zeros(SHAPE, np.uint8)
    inst = np.zeros(SHAPE, np.uint8)
    sem[:, :, :3] = 255
    sem[:, :, 3:5] = 9
    sem[100:160, 150:175, 3:6] = 11
    sem[160:, 175:, 3:5] = 17
    x0, y0 = g.integers(150, 220, 2)
    sem[x0:x0 + 30, y0 - 40:y0, 5:20] = 255
    for cls, n, (sx, sy, sz) in ((13, 2, (30, 20, 20)), (15, 2, (12, 12, 8)), (18, 3, (1, 1, 12))):
        for _ in range(n):
            x, y = g.integers(0, 250 - sx), g.integers(0, 250 - sy)
            sem[x:x + sx, y:y + sy, 5:5 + sz] = cls
    next_id = 1
    for cls, n, (sx, sy, sz) in ((1, 3, (20, 9, 7)), (6, 2, (3, 3, 9)), (2, 1, (8, 3, 6)), (4, 1, (40, 12, 14))):
        for _ in range(n):
            x, y = g.integers(0, 250 - sx), g.integers(10, 240 - sy)
            sem[x:x + sx, y:y + sy, 5:5 + sz] = cls
            if with_instances:
                inst[x:x + sx, y:y + sy, 5:5 + sz] = next_id
                next_id += 7                                   # sparse, unordered-looking ids
    return sem, inst


def points(seed):
    g = np.random.default_rng(seed)
    lo, hi = np.array([-2.0, -27.0, -3.0]), np.array([53.0, 27.0, 5.0])
    xyz = (np.round((lo + (hi - lo) * g.random((N_POINTS, 3))) * 64) / 64).astype(np.float32)   # multiples of 1/64
    xyz[:40] = (np.round(xyz[:40] / 0.2) * 0.2).astype(np.float32)          # on voxel faces
    xyz[40:44] = np.array([[0.0, -25.6, -2.0], [51.2, 25.6, 4.4], [51.19999, -25.6, 4.39999], [0.0, 0.0, 0.0]], np.float32)
    intensity = (g.integers(0, 64, (N_POINTS, 1)) / 64).astype(np.float32)
    coords = np.concatenate([xyz, intensity], 1)
    # features are copied, not computed: a pattern over (point, channel, pass) that every index error breaks and that
    # deflate stores in a few bytes
    n, c = np.arange(N_POINTS)[:, None], np.arange(V)[None, :]
    vote = (((n * 5 + c * 3 + seed) % 61) / 8 - 3).astype(np.float32)
    t, c, n = np.arange(N_TTA)[:, None, None], np.arange(E)[None, :, None], np.arange(N_POINTS)[None, None, :]
    emb = (((n * 11 + c * 37 + t * 5 + seed) % 97) / 16 - 3).astype(np.float16)
    label = (g.integers(0, 1 << 12, N_POINTS) << 16 | g.integers(0, 260, N_POINTS)).astype(np.int32)
    return {"embedding": emb, "coords": coords, "vote": vote}, label


def write_tree(root):
    files = {}

    def put(rel, data: bytes):
        path = os.path.join(root, rel)
        os.makedirs(os.path.dirname(path), exist_ok=True)
        with open(path, "wb") as fh:
            fh.write(data)
        files[rel] = data

    g = np.random.default_rng(7)
    for seq in range(11):
        s = f"{seq:02d}"
        tr = np.eye(4)[:3] + np.round(g.normal(0, 0.05, (3, 4)), 4)
        put(f"dataset/sequences/{s}/calib.txt",
            ("P0: " + " ".join(["1.0", "0", "0", "0"] * 3) + "\nTr: " + " ".join(f"{v:.6e}" for v in tr.ravel()) + "\n").encode())
        put(f"dataset/sequences/{s}/times.txt", "".join(f"{0.1 * i:.6e}\n" for i in range(12)).encode())
        put(f"dataset/sequences/{s}/poses.txt",
            "".join(" ".join(f"{v:.6e}" for v in (np.eye(4)[:3] + np.round(g.normal(0, 0.1, (3, 4)), 4)).ravel()) + "\n"
                    for _ in range(12)).encode())
    for k, ((seq, frame), with_inst) in enumerate(SCANS.items()):
        put(f"dataset/sequences/{seq}/voxels/{frame}.bin", b"")
        sem, inst = scene(100 + k, with_inst)
        put(f"preprocess/instance_labels_v2/{seq}/{frame}_1_1.pkl",
            pickle.dumps({"semantic_labels": sem, "instance_labels": inst}))
        feats, label = points(200 + k)
        put(f"preprocess/waffleiron_v2/sequences/{seq}/seg_feats_tta/{frame}.pkl", pickle.dumps(feats))
        put(f"dataset/sequences/{seq}/labels/{frame}.label", label.tobytes())
    for seq, frame in SKIPPED:
        put(f"dataset/sequences/{seq}/voxels/{frame}.bin", b"")
    put("semantic-kitti.yaml", b"learning_map:\n  0: 0\n  10: 1\n  40: 9\n")     # KittiDataset reads only this map
    return files


def mask_indices(ml, shape):
    """A mask stack → (per-cell stuff index, per-cell instance index), −1 = none, and the labels."""
    labels = ml["labels"]
    masks = ml["masks"]
    assert masks.shape[0] < 255
    stuff = np.full(shape, -1, np.int16)
    thing = np.full(shape, -1, np.int16)
    n_stuff = int(sum(int(l) not in THING_IDS for l in labels))
    # stuff masks come first and are the classes not in thing_ids; instance masks follow
    for t in range(masks.shape[0]):
        m = masks[t].numpy()
        tgt = stuff if t < n_stuff else thing
        assert (tgt[m] == -1).all()
        tgt[m] = t
    return stuff, thing, labels.numpy(), n_stuff


def narrow(a, dtype):
    """An integer array in a smaller stored type (the reference's dtype is recorded in the case's dtypes)."""
    n = a.astype(dtype)
    assert np.array_equal(n.astype(a.dtype), a)
    return n


def run_case(root, name, cfg, out):
    import pasco.data.semantic_kitti.kitti_dataset as KD

    args = {k: v for k, v in cfg.items() if k not in ("idx", "seed")}
    ds = KD.KittiDataset(root=os.path.join(root, ""), preprocess_root=os.path.join(root, "preprocess"),
                         config_path=os.path.join(root, "semantic-kitti.yaml"), **args)
    draws = {"emb": [], "crop": []}
    randint, crop = np.random.randint, KD.KittiDataset.crop

    def rec_randint(*a, **k):
        v = randint(*a, **k)
        draws["emb"].append(int(v))
        return v

    def rec_crop(*a):
        st = np.random.get_state()
        draws["crop"].append(np.random.rand(3))
        np.random.set_state(st)
        return crop(*a)

    np.random.seed(cfg["seed"])
    random.seed(cfg["seed"])
    np.random.randint, KD.KittiDataset.crop = rec_randint, staticmethod(rec_crop)
    try:
        b = ds[cfg["idx"]]
    finally:
        np.random.randint, KD.KittiDataset.crop = randint, staticmethod(crop)
    order = [next(i for i, s in enumerate(ds.scans) if s["sequence"] == q and s["frame_id"] == f)
             for q, f in zip(b["sequence"], b["frame_id"])]
    p = f"{name}/"
    meta = dict(cfg, order=order, emb=draws["emb"], frame_id=b["frame_id"], sequence=b["sequence"],
                scans=[f"{s['sequence']}/{s['frame_id']}" for s in ds.scans])
    out[p + "meta"] = np.frombuffer(json.dumps(meta).encode(), np.uint8)
    if draws["crop"]:
        out[p + "crop"] = np.stack(draws["crop"])
    out[p + "Ts"] = torch.stack(b["Ts"]).numpy()
    out[p + "global_min_Cs"], out[p + "global_max_Cs"] = b["global_min_Cs"].numpy(), b["global_max_Cs"].numpy()
    # the untransformed volumes are the scans' label pickles, stacked: checked here, not stored
    for key, pk in (("semantic_label_origin", "semantic_labels"), ("instance_label_origin", "instance_labels")):
        want = np.stack([pickle.load(open(os.path.join(root, "preprocess", "instance_labels_v2", q, f"{f}_1_1.pkl"), "rb"))[pk]
                         for q, f in zip(b["sequence"], b["frame_id"])])
        assert b[key].dtype == torch.uint8 and np.array_equal(b[key].numpy(), want), key
    for m in range(len(order)):
        q = f"{p}{m}/"
        # in_feats: the columns the reference computes (radius, xyz − voxel centre, xyz) and, for the columns it copies
        # (vote, intensity, embedding), the scan's point index of each row
        feats = b["in_feats"][m].numpy()
        with open(os.path.join(root, "preprocess/waffleiron_v2/sequences", b["sequence"][m], "seg_feats_tta",
                               f"{b['frame_id'][m]}.pkl"), "rb") as fh:
            wf = pickle.load(fh)
        xyz = wf["coords"][:, :3]
        index = {tuple(r): i for i, r in enumerate(xyz.tolist())}
        assert len(index) == len(xyz)
        rows = np.array([index[tuple(r)] for r in feats[:, -3:].tolist()], np.int64)
        assert np.array_equal(feats, np.concatenate(
            [wf["vote"][rows], wf["coords"][rows, 3:], feats[:, V + 1:V + 2],
             wf["embedding"][draws["emb"][m]].T[rows].astype(np.float32), feats[:, -6:]], 1))
        out[q + "in_feats_rows"] = narrow(rows, np.int16)
        out[q + "in_feats_own"] = np.ascontiguousarray(feats[:, OWN_COLUMNS])
        out[q + "in_coords"] = narrow(b["in_coords"][m].numpy(), np.int16)
        out[q + "min_C"], out[q + "max_C"] = b["min_Cs"][m].numpy(), b["max_Cs"][m].numpy()
        assert b["sem_labels"]["1_1"][m] is b["semantic_label"][m]           # stored once, as semantic_label
        for s in (2, 4):
            out[q + f"sem_1_{s}"] = b["sem_labels"][f"1_{s}"][m].numpy()
            out[q + f"geo_1_{s}"] = b["geo_labels"][f"1_{s}"][m].numpy()
        planes = {"volumes": [b["semantic_label"][m].numpy(), b["instance_label"][m].numpy(),
                              b["geo_labels"]["1_1"][m].numpy()], "volumes_origin": []}
        for key, vk in (("mask_label", "volumes"), ("mask_label_origin", "volumes_origin")):
            ml = b[key][m]
            stuff, thing, labels, n_stuff = mask_indices(ml, tuple(ml["masks"].shape[1:]))
            planes[vk] += [(stuff + 1).astype(np.uint8), (thing + 1).astype(np.uint8)]
            out[q + key + "_labels"] = labels
            out[q + key + "_dtypes"] = np.frombuffer(f"{ml['labels'].dtype},{ml['masks'].dtype}".encode(), np.uint8)
        planes = {k: np.stack(v) for k, v in planes.items()}
        assert all(v.dtype == np.uint8 for v in planes.values())
        out[q + "volumes"] = planes["volumes"]
        key = f"origin/{b['sequence'][m]}/{b['frame_id'][m]}"     # a function of the scan alone: stored once
        if key in out:
            assert np.array_equal(out[key], planes["volumes_origin"]), key
        out[key] = planes["volumes_origin"]
        out[q + "xyz"] = np.asarray(b["xyz"][m])
        out[q + "input_pcd_instance_label"] = narrow(b["input_pcd_instance_label"][m].numpy(), np.uint16)
    dt = {k: str(b[k][0].dtype) for k in ("in_feats", "in_coords", "semantic_label", "min_Cs", "max_Cs", "Ts")}
    dt.update({f"geo_1_{s}": str(b["geo_labels"][f"1_{s}"][0].dtype) for s in (1, 2, 4)})
    dt.update(global_min_Cs=str(b["global_min_Cs"].dtype), xyz=str(np.asarray(b["xyz"][0]).dtype),
              input_pcd_instance_label=str(b["input_pcd_instance_label"][0].dtype))
    out[p + "dtypes"] = np.frombuffer(json.dumps(dt).encode(), np.uint8)
    return b


def main():
    torch.set_num_threads(max(1, os.cpu_count() or 1))
    out = {}
    with tempfile.TemporaryDirectory() as root:
        files = write_tree(root)
        for rel, data in files.items():
            out["tree/" + rel] = np.frombuffer(data, np.uint8)
        for name, cfg in CASES.items():
            b = run_case(root, name, cfg, out)
            if name == "identity":
                for T in b["Ts"]:
                    assert torch.equal(T[:3, :3].abs(), torch.eye(3)), T
                    frac = (T[:3, 3].double() / 0.2) % 1.0
                    assert ((frac - 0.5).abs() > 0.02).all(), f"identity case: translation {T[:3, 3]} near a tie"
            print(name, [tuple(v.shape) for v in b["in_feats"]], [tuple(v.shape) for v in b["semantic_label"]],
                  b["frame_id"], b["sequence"])
    path = os.path.join(HERE, "scenes_semkitti.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path}: {os.path.getsize(path) / 1e6:.2f} MB")


if __name__ == "__main__":
    main()
