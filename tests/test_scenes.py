"""SemanticKITTI scene preparation (pasco_b200/scenes.py, csrc/scenes.cu) against the reference's own
KittiDataset.__getitem__ on a synthetic tree (tests/golden/scenes_semkitti.npz, tests/golden/make_golden_scenes.py):
the host's draws, the prepared batch field by field, the device reads, the criterion's list form and a training step."""
import json
import os
import pickle
import random
import re
import subprocess
import sys
import warnings

import numpy as np
import pytest
import torch

from pasco_b200 import _lib
from pasco_b200 import criterion as CR
from pasco_b200 import scenes as SC

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402

GOLD = "scenes_semkitti.npz"
CASES = ("train_rot", "val_tta", "no_inst", "identity")
K = 20


def _meta(g, case):
    return json.loads(bytes(g[f"{case}/meta"]).decode())


@pytest.fixture(scope="module")
def gold():
    return parity.fixture(GOLD)


@pytest.fixture(scope="module")
def tree(gold, tmp_path_factory):
    root = tmp_path_factory.mktemp("semkitti")
    for k in gold:
        if k.startswith("tree/"):
            path = root / k[len("tree/"):]
            path.parent.mkdir(parents=True, exist_ok=True)
            path.write_bytes(gold[k].tobytes())
    return str(root)


def _dataset(tree, meta, **kw):
    args = {k: meta[k] for k in ("split", "n_subnets", "data_aug", "max_angle", "translate_distance", "scale_range")}
    return SC.SemanticKittiScenes(root=tree, preprocess_root=os.path.join(tree, "preprocess"), **args, **kw)


def _raw(gold, tree, case):
    meta = _meta(gold, case)
    ds = _dataset(tree, meta)
    np.random.seed(meta["seed"])
    random.seed(meta["seed"])
    return ds, ds[meta["idx"]]


def _np_dtype(torch_dtype: str):
    return np.dtype(torch_dtype.split(".")[-1])


def _reference_case(gold, tree, case):
    """The reference's collate_fn output for a case, decoded from the fixture's stored forms (make_golden_scenes.py's
    docstring): per item, numpy arrays in the reference's dtypes, each mask stack as per-cell stuff and instance indices
    (−1 = none) with its labels; and the untransformed volumes, which are the scans' label pickles stacked."""
    meta, p = _meta(gold, case), f"{case}/"
    dt = json.loads(bytes(gold[p + "dtypes"]).decode())
    items, origin = [], {"semantic_labels": [], "instance_labels": []}
    for m, (seq, frame) in enumerate(zip(meta["sequence"], meta["frame_id"])):
        q = f"{p}{m}/"
        with open(os.path.join(tree, "preprocess/waffleiron_v2/sequences", seq, "seg_feats_tta", f"{frame}.pkl"), "rb") as fh:
            wf = pickle.load(fh)
        with open(os.path.join(tree, "preprocess/instance_labels_v2", seq, f"{frame}_1_1.pkl"), "rb") as fh:
            lab = pickle.load(fh)
        for k in origin:
            origin[k].append(lab[k].astype(np.uint8))
        rows, own = gold[q + "in_feats_rows"].astype(np.int64), gold[q + "in_feats_own"]
        feats = np.concatenate([wf["vote"][rows], wf["coords"][rows, 3:], own[:, :1],
                                wf["embedding"][meta["emb"][m]].T[rows].astype(np.float32), own[:, 1:]], 1)
        vol, org = gold[q + "volumes"], gold[f"origin/{seq}/{frame}"]
        mask = lambda key, st, th: {"stuff": st.astype(np.int16) - 1, "thing": th.astype(np.int16) - 1,  # noqa: E731
                                    "labels": gold[q + key + "_labels"],
                                    "dtypes": bytes(gold[q + key + "_dtypes"]).decode()}
        items.append({
            "in_feats": feats.astype(_np_dtype(dt["in_feats"])),
            "in_coords": gold[q + "in_coords"].astype(_np_dtype(dt["in_coords"])),
            "xyz": gold[q + "xyz"],
            "input_pcd_instance_label": gold[q + "input_pcd_instance_label"].astype(_np_dtype(dt["input_pcd_instance_label"])),
            "min_C": gold[q + "min_C"], "max_C": gold[q + "max_C"],
            "semantic_label": vol[0], "instance_label": vol[1],
            "sem_labels": {"1_1": vol[0], "1_2": gold[q + "sem_1_2"], "1_4": gold[q + "sem_1_4"]},
            "geo_labels": {"1_1": vol[2], "1_2": gold[q + "geo_1_2"], "1_4": gold[q + "geo_1_4"]},
            "mask_label": mask("mask_label", vol[3], vol[4]),
            "mask_label_origin": mask("mask_label_origin", org[0], org[1]),
        })
    return {"items": items, "dtypes": dt, "Ts": gold[p + "Ts"], "global_min_Cs": gold[p + "global_min_Cs"],
            "global_max_Cs": gold[p + "global_max_Cs"], "semantic_label_origin": np.stack(origin["semantic_labels"]),
            "instance_label_origin": np.stack(origin["instance_labels"])}


# ---- CPU ------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", CASES)
def test_draws_match_the_reference(gold, tree, case):
    meta = _meta(gold, case)
    ds, raw = _raw(gold, tree, case)
    assert [f"{s['sequence']}/{s['frame_id']}" for s in ds.scans] == meta["scans"]
    assert [r["frame_id"] for r in raw] == meta["frame_id"] and [r["sequence"] for r in raw] == meta["sequence"]
    assert [r["emb_index"] for r in raw] == meta["emb"]
    for m, r in enumerate(raw):
        assert torch.equal(r["T"], torch.from_numpy(gold[f"{case}/Ts"][m]))
        assert torch.equal(r["T_inv"], torch.inverse(r["T"]))
    if meta["split"] == "train":
        assert np.array_equal(np.stack([r["crop"] for r in raw]), gold[f"{case}/crop"])
    else:
        assert all(r["crop"] is None for r in raw)


def test_argument_checks(gold, tree):
    meta = _meta(gold, "train_rot")
    with pytest.raises(ValueError, match="n_fuse_scans"):
        _dataset(tree, meta, n_fuse_scans=2)
    _, raw = _raw(gold, tree, "train_rot")
    mixed = [raw[0], dict(raw[1], crop=None)]
    with pytest.raises(ValueError, match="all cropped"):
        SC.prepare(mixed, "cpu")
    with pytest.raises(ValueError, match="no items"):
        SC.prepare([], "cpu")


def test_stats_offsets_match_the_header():
    header = open(os.path.join(parity.ROOT, "include", "pasco_sm100.h")).read()
    for name in ("BND", "N_LABELLED", "N_INSTANCE", "SEM_EXT", "N_SEM_ROWS", "BOX", "N_SEM_KEPT", "N_POINTS",
                 "N_POINTS_KEPT", "CLS_ORIGIN", "INST_ORIGIN", "CLS", "INST", "STATS"):
        m = re.search(rf"\bPASCO_SCENE_{name} = (\d+)", header)
        assert m and int(m.group(1)) == getattr(SC, name), name


def test_scene_symbols_declared_and_kernels_use_no_local_memory():
    header = open(os.path.join(parity.ROOT, "include", "pasco_sm100.h")).read()
    names = [n for n in _lib.PROTOTYPES if n.startswith("pasco_scene_")]
    assert len(names) == 9
    for n in names:
        decl = re.search(rf"\bint {n}\(([^;]*)\);", header)
        assert decl, n
        assert decl.group(1).count(",") + 1 == len(_lib.PROTOTYPES[n][1]), n
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = [f for f in re.split(r"\n\s*Function : ", sass)[1:] if "k_scene_" in f.split("\n", 1)[0]]
    assert len(funcs) >= 12
    for f in funcs:
        assert not re.search(r"\b(LDL|STL)\b", f), f.split("\n", 1)[0]


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _near_tie(T_inv, cells, eps=1e-4):
    """Per cell (world voxel coordinates [n, 3]): whether the inverse transform's pre-rounding coordinate, in fp64, lies
    within eps of a half-integer on some axis — where the CPU's fp32 summation order can decide the rounding."""
    mb = np.array([0.0, -25.6, -2.0])
    p = cells * 0.2 + 0.1 + mb
    h = p @ T_inv[:3, :3].astype(np.float64).T + T_inv[:3, 3].astype(np.float64)
    q = (h - mb - 0.1) / 0.2
    return (np.abs(np.abs(q - np.floor(q)) - 0.5) < eps).any(1)


def _masks(ml):
    labels = ml["labels"].cpu().numpy()
    masks = ml["masks"].cpu().numpy()
    stuff = np.full(masks.shape[1:], -1, np.int16)
    thing = np.full(masks.shape[1:], -1, np.int16)
    n_stuff = int(sum(int(v) not in SC.THING_IDS for v in labels))
    for t in range(masks.shape[0]):
        (stuff if t < n_stuff else thing)[masks[t]] = t
    return stuff, thing, labels


def _compare_volume(name, got, want, allowed):
    """Bit-equal, or different only at cells flagged in `allowed`; returns the number of such cells."""
    assert got.shape == want.shape and got.dtype == want.dtype, (name, got.shape, want.shape, got.dtype, want.dtype)
    diff = got != want
    if diff.any():
        assert allowed is not None and not (diff & ~allowed).any(), (name, int(diff.sum()))
    return int(diff.sum())


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES)
def test_prepared_batch_matches_the_reference(gold, tree, case):
    _, raw = _raw(gold, tree, case)
    b = SC.prepare(raw, "cuda")
    torch.cuda.synchronize()
    ref = _reference_case(gold, tree, case)
    dt = ref["dtypes"]
    np_ = lambda t: t.cpu().numpy()  # noqa: E731
    assert np.array_equal(np_(b["global_min_Cs"]), ref["global_min_Cs"])
    assert np.array_equal(np_(b["global_max_Cs"]), ref["global_max_Cs"])
    assert str(b["global_min_Cs"].dtype) == dt["global_min_Cs"] and str(b["Ts"][0].dtype) == dt["Ts"]
    for key in ("semantic_label_origin", "instance_label_origin"):
        assert b[key].dtype == torch.uint8 and np.array_equal(np_(b[key]), ref[key]), key
    exceptions = 0
    for m, want in enumerate(ref["items"]):
        assert np.array_equal(np_(b["Ts"][m]), ref["Ts"][m])
        assert np.array_equal(np_(b["min_Cs"][m]), want["min_C"]) and np.array_equal(np_(b["max_Cs"][m]), want["max_C"])
        assert str(b["min_Cs"][m].dtype) == dt["min_Cs"] and str(b["max_Cs"][m].dtype) == dt["max_Cs"]
        size = want["semantic_label"].shape
        box = np.stack(np.meshgrid(*[np.arange(n) for n in size], indexing="ij"), -1).reshape(-1, 3) + want["min_C"]
        tie = _near_tie(raw[m]["T_inv"].numpy(), box).reshape(size)
        allowed = None if case == "identity" else tie
        for key in ("semantic_label", "instance_label"):
            exceptions += _compare_volume(key, np_(b[key][m]), want[key], allowed)
        for s in (1, 2, 4):
            blk = tie.reshape(size[0] // s, s, size[1] // s, s, size[2] // s, s).any((1, 3, 5))
            a = None if allowed is None else blk
            for key in ("sem_labels", "geo_labels"):
                exceptions += _compare_volume(f"{key} 1_{s}", np_(b[key][f"1_{s}"][m]), want[key][f"1_{s}"], a)
            assert str(b["geo_labels"][f"1_{s}"][m].dtype) == dt[f"geo_1_{s}"]
        assert b["sem_labels"]["1_1"][m] is b["semantic_label"][m]
        for key, a in (("mask_label", allowed), ("mask_label_origin", None)):
            stuff, thing, labels = _masks(b[key][m])
            w = want[key]
            assert np.array_equal(labels, w["labels"]), key
            assert w["dtypes"] == f"{b[key][m]['labels'].dtype},{b[key][m]['masks'].dtype}"
            exceptions += _compare_volume(key + " stuff", stuff, w["stuff"], a)
            exceptions += _compare_volume(key + " thing", thing, w["thing"], a)
        # points: fp32 features, int64 coordinates, fp64 xyz and the int32 point labels bit for bit
        for key in ("in_feats", "in_coords", "xyz", "input_pcd_instance_label"):
            got = np_(b[key][m])
            assert got.shape == want[key].shape and got.dtype == want[key].dtype, (key, got.shape, want[key].shape)
            assert np.array_equal(got, want[key]), (key, int((got != want[key]).sum()))
    assert b["frame_id"] == _meta(gold, case)["frame_id"] and b["sequence"] == _meta(gold, case)["sequence"]
    print(f"{case}: {exceptions} cells differ next to a rounding tie")
    if case == "identity":
        assert exceptions == 0


def _sync_count(fn):
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, [str(x.message) for x in w if "called a synchronizing" in str(x.message)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", ["train_rot", "val_tta"])
def test_prepare_reads_the_device_twice_per_item(gold, tree, case):
    _, raw = _raw(gold, tree, case)
    SC.prepare(raw, "cuda")                                      # warm the allocator: a first cudaMalloc may synchronise
    torch.cuda.synchronize()
    _, syncs = _sync_count(lambda: SC.prepare(raw, "cuda"))
    assert len(syncs) == SC.PREP_SYNCS * len(raw), syncs


@pytest.mark.gpu
def test_no_labelled_class_raises(gold, tree):
    _, raw = _raw(gold, tree, "no_inst")
    empty = dict(raw[0], semantic=np.where(raw[0]["semantic"] == 255, 255, 0).astype(np.uint8))
    with pytest.raises(ValueError, match="no labelled class"):
        SC.prepare([empty], "cuda")
    unknown = dict(raw[0], semantic=np.full_like(raw[0]["semantic"], 255))
    with pytest.raises(ValueError, match="no labelled cell"):
        SC.prepare([unknown], "cuda")


def _criterion(M, dev="cuda"):
    return CR.SetCriterion(K, [torch.ones(K + 1, device=dev)] * M, torch.ones(K, device=dev))


@pytest.mark.gpu
def test_list_form_equals_stacked_form():
    from pasco_b200.synthetic import make_scene, training_batch
    torch.manual_seed(0)
    net = parity.pasconet(M=2, f=16, num_queries=20, in_channels=16).cuda().train()
    sc = training_batch(make_scene((64, 64, 8), 0.1, 2, 16, K, seed=0, n_masks=6))
    out = net([f.cuda() for f in sc["in_feats"]], [c.cuda() for c in sc["in_coords"]], sc["global_min_Cs"],
              sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
    listed = dict(sc, semantic_label=list(sc["semantic_label"].unbind(0)),
                  sem_labels={k: list(v.unbind(0)) for k, v in sc["sem_labels"].items()},
                  geo_labels=dict(sc["geo_labels"], **{"1_1": list(sc["geo_labels"]["1_1"].unbind(0))}))
    crit = _criterion(2)
    assert CR._covered(out, sc, crit) and CR._covered(out, listed, crit)
    t0, terms0 = CR.fused_training_loss(out, sc, crit, net.class_frequencies)
    t1, terms1 = CR.fused_training_loss(out, listed, crit, net.class_frequencies)
    assert torch.equal(t0, t1) and list(terms0) == list(terms1)
    for k in terms0:
        assert torch.equal(torch.as_tensor(terms0[k]), torch.as_tensor(terms1[k])), k


@pytest.mark.gpu
def test_prepared_batch_runs_fused(gold, tree, monkeypatch):
    from pasco_b200.net3d import PascoNet
    _, raw = _raw(gold, tree, "val_tta")
    b = SC.prepare(raw, "cuda")
    assert b["semantic_label"][0].shape != b["semantic_label"][1].shape
    torch.manual_seed(0)
    net = PascoNet(n_infers=2, f=16, num_queries=20).cuda().train()
    out = net(b["in_feats"], b["in_coords"], b["global_min_Cs"], b["global_max_Cs"], b["min_Cs"], b["max_Cs"])
    crit = _criterion(2)
    assert CR._covered(out, b, crit)
    CR.fused_training_loss(out, b, crit, net.class_frequencies)   # warm the allocator
    torch.cuda.synchronize()

    def no_fallback(*a, **k):
        raise AssertionError("fell back to training_loss")
    monkeypatch.setattr(CR, "training_loss", no_fallback)
    (total, _), syncs = _sync_count(lambda: CR.fused_training_loss(out, b, crit, net.class_frequencies))
    assert len(syncs) == CR.FUSED_SYNCS, syncs
    assert torch.isfinite(total)


def _reference_batch(gold, tree, case, dev):
    """The fixture's collate_fn output on the device."""
    ref, meta = _reference_case(gold, tree, case), _meta(gold, case)
    items = ref["items"]
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(dev)  # noqa: E731
    per = lambda k: [t(it[k]) for it in items]  # noqa: E731

    def ml(w):
        masks = np.stack([(w["stuff"] == i) | (w["thing"] == i) for i in range(len(w["labels"]))])
        return {"labels": t(w["labels"]), "masks": t(masks)}
    sem = per("semantic_label")
    return {
        "frame_id": meta["frame_id"], "sequence": meta["sequence"], "xyz": [it["xyz"] for it in items],
        "geo_labels": {f"1_{s}": [t(it["geo_labels"][f"1_{s}"]) for it in items] for s in (1, 2, 4)},
        "sem_labels": dict({f"1_{s}": [t(it["sem_labels"][f"1_{s}"]) for it in items] for s in (2, 4)}, **{"1_1": sem}),
        "semantic_label": sem, "instance_label": per("instance_label"),
        "semantic_label_origin": t(ref["semantic_label_origin"]), "instance_label_origin": t(ref["instance_label_origin"]),
        "mask_label": [ml(it["mask_label"]) for it in items],
        "mask_label_origin": [ml(it["mask_label_origin"]) for it in items],
        "in_coords": per("in_coords"), "in_feats": per("in_feats"),
        "input_pcd_instance_label": per("input_pcd_instance_label"), "Ts": [t(T) for T in ref["Ts"]],
        "global_min_Cs": t(ref["global_min_Cs"]), "global_max_Cs": t(ref["global_max_Cs"]),
        "min_Cs": per("min_C"), "max_Cs": per("max_C"),
    }


@pytest.mark.gpu
def test_training_step_on_a_prepared_batch_matches_the_reference_batch(gold, tree):
    from pasco_b200 import metrics as MT
    from pasco_b200.net3d import PascoNet, evaluated_subnets
    _, raw = _raw(gold, tree, "identity")
    batches = [SC.prepare(raw, "cuda"), _reference_batch(gold, tree, "identity", "cuda")]
    results = []
    for b in batches:
        torch.manual_seed(0)
        net = PascoNet(n_infers=2, f=16, num_queries=20).cuda().train()
        evs = {i: MT.Evaluator(n_entries=1, n_classes=K, uncertainty=False) for i in evaluated_subnets(2)}
        total, terms = net.step(b, _criterion(2), net.class_frequencies, epoch=1, metrics=evs)
        total.backward()
        grads = [p.grad.clone() for p in net.parameters() if p.grad is not None]
        results.append((total.detach(), {k: torch.as_tensor(v).detach() for k, v in terms.items()}, grads,
                        {i: ev.compute() for i, ev in evs.items()}))
    (t0, k0, g0, e0), (t1, k1, g1, e1) = results
    assert torch.equal(t0, t1) and list(k0) == list(k1)
    for k in k0:
        assert torch.equal(k0[k], k1[k]), k
    assert len(g0) == len(g1) and all(torch.equal(a, b) for a, b in zip(g0, g1))
    assert repr(e0) == repr(e1)
