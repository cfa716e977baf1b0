"""criterion.fused_training_loss — the reference's training objective on the grouped setloss kernels — against the
reference's stored values (tests/golden/loss_m2.npz), against `training_loss` on the device at scale, and for its sync
budget, edge cases and fallbacks."""
import os
import re
import subprocess

import numpy as np
import pytest
import torch

from pasco_b200 import _lib
from pasco_b200 import criterion as CR

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden", "loss_m2.npz")
GROUP_SYMBOLS = ("pasco_setloss_keep_group", "pasco_setloss_match_cost_group", "pasco_setloss_pair_sums_group",
                 "pasco_setloss_pair_backward_group", "pasco_setloss_ssc_forward_group",
                 "pasco_setloss_ssc_backward_group", "pasco_lovasz_errors_group", "pasco_lovasz_grad_group",
                 "pasco_lovasz_backward_group")
LEVELS = 4


def _close(a, b, tol):
    a, b = float(a), float(b)
    if np.isnan(b):
        return np.isnan(a)
    return abs(a - b) <= tol * max(1.0, abs(b))


def _rel_l2(a, b):
    return float((a - b).norm() / b.norm().clamp(min=1e-30))


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_group_symbols_declared_and_typed():
    header = open(os.path.join(ROOT, "include", "pasco_sm100.h")).read()
    for name in GROUP_SYMBOLS:
        assert re.search(rf"\bint {name}\(", header), name
        res, args = _lib.PROTOTYPES[name]
        assert res is _lib.C.c_int and args[0] is _lib.C.c_void_p and args[1] is _lib.C.c_int32 and args[-1] is _lib.C.c_void_p
    assert _lib.C.sizeof(_lib.SetlossLevel) == 216 and _lib.C.sizeof(_lib.LovaszTerm) == 96   # the header's layout


def test_group_kernels_use_no_local_memory():
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    seen = set()
    for f in re.split(r"\n\s*Function : ", sass)[1:]:
        head = f.split("\n", 1)[0]
        m = re.search(r"(k_sl_\w+?|k_lov_\w+?)E", head)
        if m:
            seen.add(m.group(1))
            assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert "k_sl_keep" in seen and {"k_sl_cost", "k_sl_ssc_forward", "k_lov_grad"} <= seen, seen


def _gold_inputs(g, dev="cpu", M=2):
    leaves = {}

    def t(a, grad=False):
        x = torch.as_tensor(np.asarray(a)).to(dev)
        return x.clone().requires_grad_(True) if grad else x

    def leaf(name):
        leaves[name] = t(g[name], True)
        return leaves[name]
    sem_at = {s: [CR.Rows(leaf(f"sem{s}_F_m{m}"), t(g[f"sem{s}_C_m{m}"])) for m in range(M)] for s in (1, 2, 4)}
    preds = []
    for m in range(M):
        lv = [{"voxel_logits": CR.Rows(leaf(f"vox_F_m{m}_l{l}"), t(g[f"vox_C_m{m}"])), "query_logits": leaf(f"query_m{m}_l{l}")}
              for l in range(LEVELS)]
        lv[0]["aux_outputs"] = lv[1:]
        preds.append(lv[0])
    sem = t(g["semantic_label"])
    batch = {"sem_labels": {f"1_{s}": t(g[f"sem_labels_1_{s}"]) for s in (1, 2, 4)},
             "min_Cs": [torch.as_tensor(g["min_C"])] * M, "max_Cs": [torch.as_tensor(g["max_C"])] * M,
             "semantic_label": sem,
             "mask_label": [{"labels": torch.as_tensor(g["labels"][m]), "masks": t(g["masks"][m])} for m in range(M)],
             "geo_labels": {"1_1": torch.where(sem == 255, 255.0, (sem > 0).float())}}
    freqs = {f"1_{s}": g["class_frequencies"][i] for i, s in enumerate((1, 2, 4))}
    crit = CR.SetCriterion(20, list(torch.as_tensor(g["class_weights"])), torch.as_tensor(g["compl_labelweights"]))
    return {"sem_logits_at_scales": sem_at, "panop_predictions": preds}, batch, freqs, crit, leaves


def test_cpu_inputs_run_the_torch_path():
    g = dict(np.load(GOLD))
    out, batch, freqs, crit, _ = _gold_inputs(g)
    total, terms = CR.fused_training_loss(out, batch, crit, freqs)
    out2, batch2, freqs2, crit2, _ = _gold_inputs(g)
    want, want_terms = CR.training_loss(out2, batch2, crit2, freqs2)
    assert float(total.detach()) == float(want.detach()) and list(terms) == list(want_terms)


# ---- GPU ------------------------------------------------------------------------------------------------------------
class _Recording(CR.HungarianMatcher):
    """The criterion's matcher, keeping every assignment it makes (training_loss keeps only the last subnet's)."""

    def __init__(self):
        super().__init__(1.0, 20.0, 1.0)
        self.seen = []

    def __call__(self, *a):
        r = super().__call__(*a)
        self.seen.append(r)
        return r


@pytest.mark.gpu
def test_fixture_terms_assignments_and_gradients():
    g = dict(np.load(GOLD))
    out, batch, freqs, crit, leaves = _gold_inputs(g, "cuda")
    total, terms = CR.fused_training_loss(out, batch, crit, freqs)
    assert _close(total, g["total"], 1e-4), (float(total), float(g["total"]))
    for m in range(2):
        for lv in range(LEVELS):
            qi, tj = crit.subnet_indices[m][lv]
            assert np.array_equal(torch.stack([qi, tj]).numpy(), g[f"match_m{m}_l{lv}"]), (m, lv)
    for k, v in terms.items():
        if k.startswith("compl_"):
            ref = g[k.replace("_loss", "")]
        elif "_level" in k:
            ref = (g[f"{k}_m0"] + g[f"{k}_m1"]) / 2
        else:
            ref = (g[f"{k}_m0"] + g[f"{k}_m1"]) / 2
        assert _close(v, ref, 1e-4), (k, float(v), float(ref))
    total.backward()
    for name, t in leaves.items():
        if not name.startswith(("vox_F", "query", "sem")):
            continue
        ref = torch.as_tensor(g[f"grad_{name}"])
        got = t.grad.cpu() if t.grad is not None else torch.zeros_like(ref)
        scale = float(ref.abs().max())
        assert float((got - ref).abs().max()) <= 1e-3 * max(scale, 1e-12) + 1e-9, (name, scale)


def _scale_case(N=400_000, Q=100, T=30, M=2, K=20, seed=0, grid=(128, 128, 32), dev="cuda"):
    g = torch.Generator().manual_seed(seed)
    X, Y, Z = grid
    cells = torch.randperm(X * Y * Z, generator=g)[:N]
    xyz = torch.stack([cells // (Y * Z), (cells // Z) % Y, cells % Z], 1).int()
    C = torch.cat([torch.zeros(N, 1, dtype=torch.int32), xyz], 1).to(dev)
    leaves = []

    def leaf(*shape):
        t = (torch.randn(*shape, generator=g) * 2).to(dev).requires_grad_(True)
        leaves.append(t)
        return t
    sem_at = {}
    for s in (1, 2, 4):
        n = N // (s * s)
        sem_at[s] = [CR.Rows(leaf(n, K), torch.cat([torch.zeros(n, 1, dtype=torch.int32), (xyz[:n] // s) * s], 1).to(dev))
                     for _ in range(M)]
    preds = []
    for m in range(M):
        lv = [{"voxel_logits": CR.Rows(leaf(N, Q), C), "query_logits": leaf(1, Q, K + 1)} for _ in range(LEVELS)]
        lv[0]["aux_outputs"] = lv[1:]
        preds.append(lv[0])
    sem = torch.randint(0, K, (M, X, Y, Z), generator=g).to(torch.uint8)
    sem[torch.rand(sem.shape, generator=g) < 0.05] = 255
    geo = torch.where(sem == 255, 255.0, (sem > 0).float())
    masks = []
    for m in range(M):
        mk = torch.zeros(T, X, Y, Z, dtype=torch.bool)
        for i in range(T):
            lo = [int(torch.randint(0, d - d // 4, (1,), generator=g)) for d in grid]
            mk[i, lo[0]:lo[0] + X // 4, lo[1]:lo[1] + Y // 4, lo[2]:lo[2] + Z // 4] = True
        masks.append({"labels": torch.randint(1, K, (T,), generator=g).to(torch.uint8), "masks": mk.to(dev)})
    sem_labels = {f"1_{s}": sem[:, ::s, ::s, ::s].contiguous().to(dev) for s in (1, 2, 4)}
    batch = {"sem_labels": sem_labels, "min_Cs": [torch.zeros(3, dtype=torch.int64)] * M,
             "max_Cs": [torch.tensor([X - 1, Y - 1, Z - 1])] * M, "semantic_label": sem.to(dev), "mask_label": masks,
             "geo_labels": {"1_1": geo.to(dev)}}
    freqs = {f"1_{s}": np.linspace(1.0, 5.0, K) for s in (1, 2, 4)}
    cw = [torch.linspace(0.5, 1.5, K + 1) for _ in range(M)]
    crit = CR.SetCriterion(K, cw, torch.linspace(0.2, 1.0, K), matcher=_Recording())
    return {"sem_logits_at_scales": sem_at, "panop_predictions": preds}, batch, freqs, crit, leaves


def _both(case, **kw):
    """(fused total, terms, grads, assignments), (training_loss …) on the same inputs."""
    out, batch, freqs, crit, leaves = case
    res = []
    for fn in (CR.fused_training_loss, CR.training_loss):
        crit.matcher.seen = []
        tf32 = torch.backends.cuda.matmul.allow_tf32
        torch.backends.cuda.matmul.allow_tf32 = False
        try:
            total, terms = fn(out, batch, crit, freqs, **kw)
        finally:
            torch.backends.cuda.matmul.allow_tf32 = tf32
        grads = torch.autograd.grad(total, leaves, allow_unused=True, retain_graph=False) if total.requires_grad else []
        idx = ([a for sub in crit.subnet_indices for a in sub] if fn is CR.fused_training_loss
               else list(crit.matcher.seen))
        res.append((total, terms, grads, idx))
    return res


@pytest.mark.gpu
def test_at_scale_against_training_loss():
    case = _scale_case()
    (t1, terms1, g1, idx1), (t0, terms0, g0, idx0) = _both(case)
    assert list(terms1) == list(terms0)
    assert len(idx1) == len(idx0) == 2 * LEVELS
    for (a, b), (c, d) in zip(idx1, idx0):
        assert torch.equal(a, c) and torch.equal(b, d)
    for k in terms0:
        assert _close(terms1[k], terms0[k], 1e-5), (k, float(terms1[k]), float(terms0[k]))
    for a, b in zip(g1, g0):
        if b is not None:
            assert a is not None and _rel_l2(a, b) <= 1e-4, _rel_l2(a, b)
    # two repeat calls give the same bits
    out, batch, freqs, crit, leaves = case
    again = CR.fused_training_loss(out, batch, crit, freqs)[1]
    first = CR.fused_training_loss(out, batch, crit, freqs)[1]
    assert all(torch.equal(again[k], first[k]) for k in first)


@pytest.mark.gpu
def test_grouped_launch_equals_one_launch_per_level():
    from pasco_b200 import ops
    out, batch, freqs, crit, _ = _scale_case(N=50_000)
    dev = torch.device("cuda")
    levels = []
    for m, pred in enumerate(out["panop_predictions"]):
        bits, flags, lab, stats = ops.setloss_sample(pred["voxel_logits"].C, torch.zeros(3, dtype=torch.int32, device=dev),
                                                     batch["mask_label"][m]["masks"], batch["geo_labels"]["1_1"][m] == 255,
                                                     batch["semantic_label"][m], 20)
        ids = batch["mask_label"][m]["labels"].to(dev, torch.int32)
        for lv in [pred] + pred["aux_outputs"]:
            levels.append(dict(F=lv["voxel_logits"].F.detach().contiguous(), T=30, bits=bits, flags=flags, stats=stats,
                               query_logits=lv["query_logits"][0].detach().contiguous(), ids=ids,
                               class_weight=torch.ones(21, device=dev), lab=lab))
    grouped = ops.match_cost_group(levels, 20.0, 1.0, 1.0)
    single = torch.cat([ops.match_cost_group([lv], 20.0, 1.0, 1.0) for lv in levels])
    assert torch.equal(grouped, single)
    # matched-pair sums, forward and backward: the assignment of level l is the identity on its first T queries
    meta = [(lv["bits"], 30, lv["flags"], torch.arange(30, dtype=torch.int32, device=dev),
             torch.arange(30, dtype=torch.int32, device=dev).flip(0).contiguous()) for lv in levels]
    Fs = [lv["F"].clone().requires_grad_(True) for lv in levels]
    grouped = ops.PairSumsGroup.apply(meta, *Fs)
    g = torch.randn_like(grouped)
    g_grouped = torch.autograd.grad(grouped, Fs, g)
    for i in range(len(levels)):
        one = ops.PairSumsGroup.apply([meta[i]], Fs[i])
        assert torch.equal(one, grouped[30 * i:30 * (i + 1)])
        assert torch.equal(torch.autograd.grad(one, [Fs[i]], g[30 * i:30 * (i + 1)])[0], g_grouped[i])
    keep, kept = ops.setloss_keep_group([lv["query_logits"] for lv in levels])
    for i, lv in enumerate(levels):
        want = torch.nonzero(lv["query_logits"].argmax(-1) != 20).flatten()
        assert torch.equal(keep[i, :int(kept[i])].long(), want)
    kq = kept.tolist()
    meta = [(keep[i], min(kq[i], 128)) for i in range(len(levels)) if kq[i]]
    use = [lv for i, lv in enumerate(levels) if kq[i]]
    Fs, qs = [lv["F"] for lv in use], [lv["query_logits"] for lv in use]
    grouped = ops.SscLogitsGroup.apply(meta, *Fs, *qs)
    for i, lv in enumerate(use):
        assert torch.equal(grouped[i], ops.SscLogitsGroup.apply([meta[i]], Fs[i], qs[i])[0])
    labels = [lv["lab"] for lv in use]
    per = ops.LovaszGroup.apply(labels, *grouped)
    one = torch.cat([ops.LovaszGroup.apply([lab], x) for lab, x in zip(labels, grouped)])
    assert torch.equal(per, one)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_one_host_sync_per_call(M):
    import warnings
    out, batch, freqs, crit, _ = _scale_case(N=60_000, M=M)
    CR.fused_training_loss(out, batch, crit, freqs)            # warm the allocator: a first cudaMalloc may synchronise
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            total, _ = CR.fused_training_loss(out, batch, crit, freqs)
        finally:
            torch.cuda.set_sync_debug_mode("default")
    syncs = [str(x.message) for x in w if "called a synchronizing" in str(x.message)]
    assert len(syncs) == CR.FUSED_SYNCS, syncs


def _agree(case, **kw):
    (t1, terms1, g1, _), (t0, terms0, g0, _) = _both(case, **kw)
    assert list(terms1) == list(terms0)
    for k in terms0:
        assert _close(terms1[k], terms0[k], 1e-5), (k, float(terms1[k]), float(terms0[k]))
    for a, b in zip(g1, g0):
        if b is not None and torch.isfinite(b).all():
            assert a is not None and _rel_l2(a, b) <= 1e-4


@pytest.mark.gpu
def test_edge_cases_match_training_loss():
    # a level with no kept query: every query's arg-max is the no-object class
    case = _scale_case(N=20_000)
    with torch.no_grad():
        case[0]["panop_predictions"][0]["aux_outputs"][1]["query_logits"][..., -1] += 100.0
    _agree(case)
    # a completion pair with no row in bounds: subnet 1's bounds exclude every row
    case = _scale_case(N=20_000)
    case[1]["min_Cs"] = [case[1]["min_Cs"][0], torch.tensor([500, 500, 500])]
    case[1]["max_Cs"] = [case[1]["max_Cs"][0], torch.tensor([600, 600, 600])]
    case[0]["panop_predictions"] = case[0]["panop_predictions"][:1]
    _agree(case)
    # T = 0
    case = _scale_case(N=20_000, T=0, M=1)
    _agree(case)


@pytest.mark.gpu
@pytest.mark.parametrize("what", ["classes", "kept", "unlabelled", "rows_outside", "labels_outside", "cpu", "aux_rows",
                                  "half_queries"])
def test_fallbacks_run_training_loss(what, monkeypatch):
    case = _scale_case(N=20_000, M=1, Q=200 if what == "kept" else 100, K=70 if what == "classes" else 20)
    out, batch, freqs, crit, _ = case
    if what == "kept":
        with torch.no_grad():
            for lv in [out["panop_predictions"][0]] + out["panop_predictions"][0]["aux_outputs"]:
                lv["query_logits"][..., 0] += 100.0
    elif what == "unlabelled":
        batch["semantic_label"] = torch.full_like(batch["semantic_label"], 255)
    elif what == "rows_outside":
        C = out["panop_predictions"][0]["voxel_logits"].C.clone()
        C[0, 1] = 1000
        for lv in [out["panop_predictions"][0]] + out["panop_predictions"][0]["aux_outputs"]:
            lv["voxel_logits"] = CR.Rows(lv["voxel_logits"].F, C)
    elif what == "labels_outside":
        batch["semantic_label"] = batch["semantic_label"].clone()
        x, y, z = out["panop_predictions"][0]["voxel_logits"].C[0, 1:].tolist()
        batch["semantic_label"][0, x, y, z] = 40                 # a class id outside [0, K) at a row's cell
    elif what == "aux_rows":                                 # an aux level on the main level's rows, permuted
        aux = out["panop_predictions"][0]["aux_outputs"][0]
        aux["voxel_logits"] = CR.Rows(aux["voxel_logits"].F, aux["voxel_logits"].C.flip(0).contiguous())
    elif what == "half_queries":
        aux = out["panop_predictions"][0]["aux_outputs"][0]
        aux["query_logits"] = aux["query_logits"].detach().half()
    elif what == "cpu":
        batch["semantic_label"] = batch["semantic_label"].cpu()
    runs = []
    real = CR.training_loss

    def spy(*a, **k):
        runs.append(1)
        if what in ("rows_outside", "labels_outside", "half_queries"):   # the torch path would index outside the
            # volume, or mix fp16 query logits with fp32 class weights
            return torch.zeros(()), {}
        return real(*a, **k)
    monkeypatch.setattr(CR, "training_loss", spy)
    total, terms = CR.fused_training_loss(out, batch, crit, freqs)
    assert runs == [1], what
    if what in ("classes", "kept"):
        monkeypatch.setattr(CR, "training_loss", real)
        want, want_terms = real(out, batch, crit, freqs)
        assert float(total) == float(want) and list(terms) == list(want_terms)


@pytest.mark.gpu
def test_pasconet_end_to_end():
    from pasco_b200.net3d import PascoNet
    from pasco_b200.synthetic import make_scene, training_batch
    dev = torch.device("cuda")
    torch.manual_seed(0)
    net = PascoNet(n_classes=20, n_infers=2, in_channels=16, f=16, num_queries=20).to(dev).train()
    sc = training_batch(make_scene((64, 64, 8), 0.1, 2, 16, 20, seed=0, n_masks=6))
    out = net([f.to(dev) for f in sc["in_feats"]], [c.to(dev) for c in sc["in_coords"]], sc["global_min_Cs"],
              sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
    crit = CR.SetCriterion(20, [torch.ones(21)] * 2, torch.ones(20), matcher=_Recording())
    params = [p for p in net.parameters() if p.requires_grad]
    res = []
    for fn in (CR.fused_training_loss, CR.training_loss):
        total, _ = fn(out, sc, crit, net.class_frequencies)
        res.append((total, torch.autograd.grad(total, params, retain_graph=True, allow_unused=True)))
    (t1, g1), (t0, g0) = res
    assert _close(t1, t0, 1e-5), (float(t1), float(t0))
    a = torch.cat([x.flatten() for x, y in zip(g1, g0) if y is not None])
    b = torch.cat([y.flatten() for y in g0 if y is not None])
    assert _rel_l2(a, b) <= 1e-4, _rel_l2(a, b)
