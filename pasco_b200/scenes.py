"""SemanticKITTI scenes for PascoNet: file reading and random draws on the host, everything else on the device.

`SemanticKittiScenes` is the host half of the reference's `KittiDataset.__getitem__`
(pasco/data/semantic_kitti/kitti_dataset.py:126-490): it lists the scans, reads a scan's label pickle, WaffleIron
pickle and point labels, and makes the reference's random draws in the reference's order — `np.random.choice` of the
other items and `random.shuffle`, then per item the embedding index, `generate_random_transformation` and the crop's
`np.random.rand(3)` — so that under the same `np.random` / `random` seeds it draws the same scenes, poses and crops.
An item is a list of M raw host items; it is safe to produce in DataLoader workers (no CUDA).

`prepare(raw_items, device)` is the device half (csrc/scenes.cu): the resampling under T, the crop, the item box,
the multi-scale labels, the mask labels, the point features and `collate_fn`'s fields, with the reference's dtypes,
shapes and bits.  Per-item volumes are lists, as `collate_fn` returns them.  It reads the device PREP_SYNCS times per
item and not in the collate.
"""
from __future__ import annotations

import ctypes as C
import glob
import os
import pickle
import random
from typing import Dict, List, Sequence

import numpy as np
import torch
from scipy.spatial.transform import Rotation

from . import ops
from ._lib import ptr
from .predict import THING_IDS, step_box

PREP_SYNCS = 2          # device reads per item in prepare(): the transformed box, then the cropped box and its ids
SCALES = (1, 2, 4)

# offsets into the int32 stats block of one item (include/pasco_sm100.h, PASCO_SCENE_*)
BND, N_LABELLED, N_INSTANCE, SEM_EXT, N_SEM_ROWS, BOX, N_SEM_KEPT, N_POINTS, N_POINTS_KEPT = 0, 6, 7, 8, 14, 16, 22, 23, 24
CLS_ORIGIN, INST_ORIGIN, CLS, INST, STATS = 256, 512, 768, 1024, 1280

SPLITS = {
    "train": ["00", "01", "02", "03", "04", "05", "06", "07", "09", "10"],
    "val": ["08"],
    "test": ["11", "12", "13", "14", "15", "16", "17", "18", "19", "20", "21"],
    "trainval": ["00", "01", "02", "03", "04", "05", "06", "07", "08", "09", "10"],
}


def random_transformation(max_angle, scale_range, max_translation) -> torch.Tensor:
    """transform_utils.generate_random_transformation(flip=True): its draws in its order, T_scale @ T @ T_flip in fp32."""
    translation = (np.random.rand(3) - 0.5) * max_translation
    rot = (np.random.rand() - 0.5) * max_angle * 2
    flip_dim = 1 if np.random.rand() > 0.5 else None
    scale = 1.0 + (np.random.rand(3) - 0.5) * scale_range
    T_flip = np.identity(4)
    if flip_dim is not None:
        T_flip[flip_dim, flip_dim] = -1
    T = np.identity(4)
    T[:3, :3] = Rotation.from_euler("xyz", [0, 0, rot], degrees=True).as_matrix()
    T[:3, 3] = translation
    T_scale = np.identity(4)
    T_scale[[0, 1, 2], [0, 1, 2]] *= scale
    f = lambda a: torch.from_numpy(a).float()  # noqa: E731
    return f(T_scale) @ f(T) @ f(T_flip)


class SemanticKittiScenes(torch.utils.data.Dataset):
    """The scans of one SemanticKITTI split; item idx = the M raw items of one MIMO batch (see the module docstring).

    Reads `<root>/dataset/sequences/<seq>/{voxels/*.bin, calib.txt, times.txt, poses.txt, labels/<frame>.label}`,
    `<preprocess_root>/instance_labels_v2/<seq>/<frame>_1_1.pkl` and
    `<preprocess_root>/waffleiron_v2/sequences/<seq>/seg_feats_tta/<frame>.pkl` (`embedding`, `coords`, `vote`)."""

    def __init__(self, split, root, preprocess_root, n_subnets=2, data_aug=False, max_angle=90.0,
                 translate_distance=0.2, scale_range=0, max_items=None, n_fuse_scans=1, complete_scale=8,
                 frame_interval=5):
        if n_fuse_scans != 1:
            raise ValueError(f"SemanticKittiScenes: n_fuse_scans must be 1 (got {n_fuse_scans}); the reference's "
                             "multi-scan branch cannot run")
        if complete_scale != 8:
            raise ValueError(f"SemanticKittiScenes: complete_scale must be 8, the scale PascoNet's boxes use "
                             f"(got {complete_scale})")
        super().__init__()
        self.split, self.root, self.preprocess_root = split, root, preprocess_root
        self.n_subnets, self.data_aug = n_subnets, data_aug
        self.max_angle, self.scale_range = max_angle, scale_range
        self.max_translation = np.array([3.0, 3.0, 2.0]) * translate_distance
        self.complete_scale = complete_scale
        self.scans = []
        for sequence in SPLITS[split]:
            for voxel_path in glob.glob(os.path.join(root, "dataset", "sequences", sequence, "voxels", "*.bin")):
                frame_id = os.path.splitext(os.path.basename(voxel_path))[0]
                if float(frame_id) % frame_interval != 0:
                    continue
                self.scans.append({"sequence": sequence, "frame_id": frame_id})
        self.scans.sort(key=lambda x: x["frame_id"])
        if max_items is not None:
            self.scans = self.scans[:max_items]
        self.calibrations, self.times, self.poses = [], [], []
        for seq in range(0, 11):
            folder = os.path.join(root, "dataset", "sequences", str(seq).zfill(2))
            self.calibrations.append(_parse_calibration(os.path.join(folder, "calib.txt")))
            self.times.append(np.loadtxt(os.path.join(folder, "times.txt"), dtype=np.float32))
            poses = _parse_poses(os.path.join(folder, "poses.txt"), self.calibrations[-1])
            self.poses.append([p.astype(np.float32) for p in poses])

    def __len__(self):
        return len(self.scans)

    def __getitem__(self, idx) -> List[Dict]:
        if self.split == "val":
            idx_list = [idx] * self.n_subnets
        else:
            idx_list = np.random.choice(len(self.scans), self.n_subnets - 1, replace=False).tolist() + [idx]
        random.shuffle(idx_list)
        return [self.raw_item(i) for i in idx_list]

    def raw_item(self, idx) -> Dict:
        """One scan's files and its draws: the embedding index, T (and T⁻¹) and the crop's np.random.rand(3)."""
        scan = self.scans[idx]
        sequence, frame_id = scan["sequence"], scan["frame_id"]
        with open(os.path.join(self.preprocess_root, "instance_labels_v2", sequence, f"{frame_id}_1_1.pkl"), "rb") as fh:
            data = pickle.load(fh)
        semantic = np.ascontiguousarray(data["semantic_labels"].astype(np.uint8))
        instance = np.ascontiguousarray(data["instance_labels"].astype(np.uint8))
        path = os.path.join(self.preprocess_root, "waffleiron_v2/sequences", sequence, "seg_feats_tta", f"{frame_id}.pkl")
        if not os.path.exists(path):
            raise FileNotFoundError(path)
        with open(path, "rb") as fh:
            feats = pickle.load(fh)
        embedding = feats["embedding"]
        emb_index = np.random.randint(0, embedding.shape[0])
        points = feats["coords"]
        if points.dtype != np.float32 or points.ndim != 2 or points.shape[1] < 3:
            raise ValueError(f"{path}: coords must be float32 [N, >= 3] (got {points.dtype} {points.shape})")
        label_path = os.path.join(self.root, "dataset", "sequences", sequence, "labels", f"{frame_id}.label")
        label = np.fromfile(label_path, dtype=np.int32)
        if self.data_aug:
            T = random_transformation(self.max_angle, self.scale_range, self.max_translation)
        else:
            T = torch.eye(4)
        crop = np.random.rand(3) if self.split == "train" else None
        # the reference concatenates these in fp32 (fp64 inputs round once, in its final .float())
        return {"sequence": sequence, "frame_id": frame_id, "semantic": semantic, "instance": instance,
                "points": np.ascontiguousarray(points), "vote": np.ascontiguousarray(feats["vote"], dtype=np.float32),
                "embedding": np.ascontiguousarray(embedding[emb_index], dtype=np.float32), "emb_index": emb_index,
                "label": label, "T": T, "T_inv": torch.inverse(T), "crop": crop}


def _parse_calibration(filename):
    calib = {}
    with open(filename) as fh:
        for line in fh:
            key, content = line.strip().split(":")
            values = [float(v) for v in content.strip().split()]
            pose = np.zeros((4, 4))
            pose[0, 0:4], pose[1, 0:4], pose[2, 0:4] = values[0:4], values[4:8], values[8:12]
            pose[3, 3] = 1.0
            calib[key] = pose
    return calib


def _parse_poses(filename, calibration):
    Tr = calibration["Tr"]
    Tr_inv = np.linalg.inv(Tr)
    poses = []
    with open(filename) as fh:
        for line in fh:
            values = [float(v) for v in line.strip().split()]
            pose = np.zeros((4, 4))
            pose[0, 0:4], pose[1, 0:4], pose[2, 0:4] = values[0:4], values[4:8], values[8:12]
            pose[3, 3] = 1.0
            poses.append(np.matmul(Tr_inv, np.matmul(pose, Tr)))
    return poses


# ------------------------------------------------------------------------------------------------
# device half
# ------------------------------------------------------------------------------------------------
def _up(a, dev, dtype=None) -> torch.Tensor:
    """Host array → device without a synchronisation (an asynchronous copy from pageable memory is staged before the
    call returns)."""
    t = a if torch.is_tensor(a) else torch.from_numpy(np.ascontiguousarray(a))
    return t.to(dev, dtype=dtype, non_blocking=True)


def _f16(T: torch.Tensor):
    return (C.c_float * 16)(*T.reshape(-1).tolist())


def _i3(v):
    return (C.c_int32 * 3)(*[int(x) for x in v])


def _mask_label(sem, inst, cls_flags, inst_flags, dev, what):
    """prepare_mask_label on the device from the volumes' present classes / ids (host flags): stuff classes ascending,
    then instance ids ascending."""
    classes = [c for c in range(256) if cls_flags[c] and c not in (0, 255)]
    if not classes:
        raise ValueError(f"prepare: {what} has no labelled class (the reference's torch.stack([]) raises here)")
    stuff = [c for c in classes if c not in THING_IDS]
    ids = [i for i in range(1, 256) if inst_flags[i]]
    slot = np.full(512, -1, np.int32)
    slot[stuff] = np.arange(len(stuff))
    slot[[256 + i for i in ids]] = len(stuff) + np.arange(len(ids))
    T = len(stuff) + len(ids)
    masks = torch.empty((T,) + tuple(sem.shape), dtype=torch.bool, device=dev)
    labels = torch.empty(T, dtype=torch.uint8, device=dev)
    ops.call("pasco_scene_masks", ptr(sem), ptr(inst), sem.numel(), ptr(_up(slot, dev)), T, ptr(masks), ptr(labels))
    return {"labels": labels, "masks": masks}


def _prepare_item(raw: Dict, train: bool, sem_o: torch.Tensor, inst_o: torch.Tensor, dev) -> Dict:
    X, Y, Z = sem_o.shape
    sem_o.copy_(torch.from_numpy(raw["semantic"]), non_blocking=True)
    inst_o.copy_(torch.from_numpy(raw["instance"]), non_blocking=True)
    T, Ti = _f16(raw["T"]), _f16(raw["T_inv"])
    stats = torch.empty(STATS, dtype=torch.int32, device=dev)
    ops.call("pasco_scene_source", ptr(sem_o), ptr(inst_o), X, Y, Z, T, ptr(stats))
    st = stats.cpu().numpy()                                                     # device read 1
    if st[N_LABELLED] == 0:
        raise ValueError(f"prepare: scan {raw['sequence']}/{raw['frame_id']} has no labelled cell")
    mask_origin = _mask_label(sem_o, inst_o, st[CLS_ORIGIN:CLS_ORIGIN + 256], st[INST_ORIGIN:INST_ORIGIN + 256], dev,
                              f"scan {raw['sequence']}/{raw['frame_id']}")
    lo = st[BND:BND + 3]
    G = st[BND + 3:BND + 6] - lo + 1
    with_inst = int(st[N_INSTANCE] > 0)
    gs = torch.empty(tuple(int(g) for g in G), dtype=torch.uint8, device=dev)
    gi = torch.empty_like(gs) if with_inst else None
    ops.call("pasco_scene_resample", ptr(sem_o), ptr(inst_o), X, Y, Z, Ti, _i3(lo), _i3(G), with_inst, ptr(gs), ptr(gi),
             ptr(stats))
    bounds = torch.empty(4, dtype=torch.float64, device=dev)
    draw = (C.c_double * 3)(*raw["crop"]) if train else None
    ops.call("pasco_scene_crop", ptr(stats), draw, int(train), ptr(bounds))
    ops.call("pasco_scene_crop_stats", ptr(gs), ptr(gi), _i3(lo), _i3(G), with_inst, ptr(bounds), ptr(stats))
    pts = _up(raw["points"], dev)
    N, pitch = pts.shape
    ext, keep = (torch.empty(N, dtype=torch.uint8, device=dev) for _ in range(2))
    ops.call("pasco_scene_points", ptr(pts), N, pitch, T, ptr(bounds), ptr(ext), ptr(keep), ptr(stats))
    st = stats.cpu().numpy()                                                     # device read 2
    if st[N_SEM_KEPT] == 0:
        raise ValueError(f"prepare: scan {raw['sequence']}/{raw['frame_id']} keeps no semantic row")

    # the item box: min_C = floor(min / 8) * 8 over the kept rows, max_C their max, compute_scene_size(·, ·, 8)
    min_C = [int(v) // 8 * 8 for v in st[BOX:BOX + 3]]
    max_C = [int(v) for v in st[BOX + 3:BOX + 6]]
    size = step_box(min_C, max_C)[2]
    sem = torch.empty(size, dtype=torch.uint8, device=dev)
    inst, geo = torch.empty_like(sem), torch.empty_like(sem)
    ops.call("pasco_scene_box", ptr(gs), ptr(gi), _i3(lo), _i3(G), with_inst, ptr(bounds), _i3(min_C), _i3(size),
             ptr(sem), ptr(inst), ptr(geo))
    sem_labels, geo_labels = {"1_1": sem}, {"1_1": geo}
    for s in SCALES[1:]:
        sz = tuple(v // s for v in size)
        sl, gl = torch.empty(sz, dtype=torch.uint8, device=dev), torch.empty(sz, dtype=torch.uint8, device=dev)
        ops.call("pasco_scene_scale", ptr(sem), *size, s, ptr(sl), ptr(gl))
        sem_labels[f"1_{s}"], geo_labels[f"1_{s}"] = sl, gl
    mask = _mask_label(sem, inst, st[CLS:CLS + 256], st[INST:INST + 256], dev,
                       f"the transformed scan {raw['sequence']}/{raw['frame_id']}")

    n_ext, n_keep = int(st[N_POINTS]), int(st[N_POINTS_KEPT])
    ext_rows = ops.compact(ext, n_ext)[0]
    keep_rows = ops.compact(keep, n_keep)[0]
    vote, emb = _up(raw["vote"], dev), _up(raw["embedding"], dev)
    V, E = vote.shape[1], emb.shape[0]
    if vote.shape[0] != N or emb.shape[1] != N or raw["label"].shape[0] != N:
        raise ValueError(f"prepare: scan {raw['sequence']}/{raw['frame_id']}: {N} points but vote {tuple(vote.shape)}, "
                         f"embedding {tuple(emb.shape)} and {raw['label'].shape[0]} point labels")
    label = _up(raw["label"], dev)
    feats = torch.empty(n_keep, V + pitch - 3 + 1 + E + 6, dtype=torch.float32, device=dev)
    coords = torch.empty(n_keep, 3, dtype=torch.int64, device=dev)
    xyz = torch.empty(n_ext, 3, dtype=torch.float64, device=dev)
    pcd_label = torch.empty(n_ext, 1, dtype=torch.int32, device=dev)
    ops.call("pasco_scene_point_rows", ptr(pts), pitch, ptr(vote), V, ptr(emb), E, N, ptr(keep_rows), n_keep, T,
             ptr(feats), ptr(coords), ptr(label), ptr(ext_rows), n_ext, ptr(xyz), ptr(pcd_label))
    return {"frame_id": raw["frame_id"], "sequence": raw["sequence"], "in_feat": feats, "in_coord": coords,
            "T": _up(raw["T"], dev), "min_C": min_C, "max_C": max_C, "semantic_label": sem, "instance_label": inst,
            "mask_label": mask, "geo_labels": geo_labels, "sem_labels": sem_labels, "mask_label_origin": mask_origin,
            "input_pcd_instance_label": pcd_label, "xyz": xyz}


def prepare(raw_items: Sequence[Dict], device) -> Dict:
    """The batch `collate_fn(items, 8)` returns for the items KittiDataset.get_individual makes from `raw_items`
    (one SemanticKittiScenes item), on `device`: same keys, dtypes, shapes and values."""
    dev = torch.device(device)
    if not raw_items:
        raise ValueError("prepare: no items")
    train = raw_items[0]["crop"] is not None
    if any((r["crop"] is not None) != train for r in raw_items):
        raise ValueError("prepare: the items of a batch are either all cropped (train) or none")
    shape = raw_items[0]["semantic"].shape
    if any(r["semantic"].shape != shape or r["instance"].shape != shape for r in raw_items):
        raise ValueError("prepare: every scan's label volumes must have one shape (collate_fn stacks them)")
    M = len(raw_items)
    sem_o = torch.empty((M,) + shape, dtype=torch.uint8, device=dev)
    inst_o = torch.empty_like(sem_o)
    items = [_prepare_item(r, train, sem_o[m], inst_o[m], dev) for m, r in enumerate(raw_items)]

    # collate_fn: the global box from the items' boxes, known on the host since each item's second read
    g_min = [min(it["min_C"][a] for it in items) for a in range(3)]
    g_max = [max(it["max_C"][a] for it in items) for a in range(3)]
    size = step_box(g_min, g_max)[2]
    i32 = lambda v: _up(torch.tensor(v, dtype=torch.int32), dev)  # noqa: E731
    per = lambda k: [it[k] for it in items]  # noqa: E731
    return {
        "frame_id": per("frame_id"), "xyz": per("xyz"),
        "geo_labels": {f"1_{s}": [it["geo_labels"][f"1_{s}"] for it in items] for s in SCALES},
        "sem_labels": {f"1_{s}": [it["sem_labels"][f"1_{s}"] for it in items] for s in SCALES},
        "sequence": per("sequence"), "semantic_label": per("semantic_label"), "instance_label": per("instance_label"),
        "semantic_label_origin": sem_o, "instance_label_origin": inst_o,
        "mask_label": per("mask_label"), "mask_label_origin": per("mask_label_origin"),
        "in_coords": per("in_coord"), "in_feats": per("in_feat"),
        "input_pcd_instance_label": per("input_pcd_instance_label"), "Ts": per("T"),
        "global_min_Cs": i32(g_min), "global_max_Cs": i32([g + s - 1 for g, s in zip(g_min, size)]),
        "min_Cs": [i32(it["min_C"]) for it in items], "max_Cs": [i32(it["max_C"]) for it in items],
    }
