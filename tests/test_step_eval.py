"""Net.step's per-step evaluation and semantic pre-training gate for PascoNet: predict.step_entries + metrics.Evaluator
against the reference's own panoptic_inference / prune_outside_coords / evaluate_all (tests/golden/step_eval_m2.npz,
tests/golden/make_golden_step_eval.py), PascoNet.step against fused_training_loss, the gate, the sync budget, and the
unmodified reference's Net.step on the drop-in."""
import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

from pasco_b200 import _lib
from pasco_b200 import criterion as CR
from pasco_b200 import metrics as MT
from pasco_b200 import predict as PR
from pasco_b200.net3d import PRETRAIN_SEM_EPOCHS, evaluated_subnets, sem_pretraining

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402

K, M, STEPS = 20, 2, 2
GOLD = "step_eval_m2.npz"


def _case(g, step, dev="cpu"):
    """(out, batch) of one step of the fixture: a training forward output and the reference's batch fields."""
    t = lambda a: torch.as_tensor(np.asarray(a)).to(dev)  # noqa: E731
    F = lambda k: t(g[k].astype(np.float32) / 16)         # noqa: E731  logits: int8 counts of 1/16
    C = lambda k: t(g[k].astype(np.int32))                # noqa: E731  coordinates: int8
    preds = [{"voxel_logits": CR.Rows(F(f"s{step}m{m}_vox_F"), C(f"s{step}m{m}_vox_C")),
              "query_logits": t(g[f"s{step}m{m}_query"])} for m in range(M)]
    sems = [CR.Rows(F(f"s{step}m{m}_sem_F"), C(f"s{step}m{m}_sem_C")) for m in range(M)]
    batch = {"min_Cs": [torch.as_tensor(g["min_C"])] * M, "max_Cs": [torch.as_tensor(g["max_C"])] * M,
             "semantic_label": torch.stack([t(g[f"s{step}m{m}_label"]) for m in range(M)]),
             "mask_label": [{"labels": t(g[f"s{step}m{m}_labels"]), "masks": t(g[f"s{step}m{m}_masks"])}
                            for m in range(M)]}
    return {"panop_predictions": preds, "sem_logits_at_scales": {1: sems}}, batch


# ---- CPU ------------------------------------------------------------------------------------------------------------
def test_box_symbol_declared_and_kernel_uses_no_local_memory():
    header = open(os.path.join(parity.ROOT, "include", "pasco_sm100.h")).read()
    assert re.search(r"\bint pasco_box_cells\(", header)
    res, args = _lib.PROTOTYPES["pasco_box_cells"]
    assert res is _lib.C.c_int and len(args) == 11
    if not os.path.exists(_lib.LIB_PATH):
        pytest.skip("library not built")
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    funcs = [f for f in re.split(r"\n\s*Function : ", sass)[1:] if "k_box_cells" in f.split("\n", 1)[0]]
    assert len(funcs) == 1
    assert not re.search(r"\b(LDL|STL)\b", funcs[0])


def test_pretraining_gate_epochs():
    # net_panoptic_sparse.py:93-98 and 337-339: pretrain_sem_epoch 2 at M = 4, 1 at M = 3, else 0; gate only for M > 2
    assert PRETRAIN_SEM_EPOCHS == {3: 1, 4: 2}
    want = {(1, 0): False, (2, 0): False, (2, 5): False, (3, 0): True, (3, 1): False, (3, 2): False, (4, 0): True,
            (4, 1): True, (4, 2): False, (5, 0): False, (8, 0): False}
    for (n, epoch), closed in want.items():
        assert sem_pretraining(n, epoch) is closed, (n, epoch)
    assert evaluated_subnets(1) == [0] and evaluated_subnets(2) == [0, 1] and evaluated_subnets(4) == [0, 3]


def test_step_box_is_compute_scene_size():
    lo, hi, size = PR.step_box(torch.tensor([8, -4, 0]), torch.tensor([35, 15, 11]))
    assert lo == (8, -4, 0) and hi == (35, 15, 11) and size == (32, 24, 16)
    assert PR.step_box(torch.tensor([0, 0, 0]), torch.tensor([63, 63, 7]))[2] == (64, 64, 8)
    with pytest.raises(ValueError, match="empty box"):
        PR.step_box(torch.tensor([5, 0, 0]), torch.tensor([-20, 3, 3]))


def test_step_entries_argument_checks():
    g = parity.fixture(GOLD)
    out, batch = _case(g, 1)
    for bad in ([2], [-1], [0, 5], [True], [0.0]):
        with pytest.raises(ValueError, match="not indices"):
            PR.step_entries(out, batch, bad)
    assert PR.step_entries(out, batch, []) == []
    wrong = dict(batch, semantic_label=batch["semantic_label"][:, :, :, :8])           # not the box's shape
    with pytest.raises(ValueError, match=r"semantic_label has shape \(32, 24, 8\), the box .* is \[32, 24, 16\]"):
        PR.step_entries(out, wrong, [1])
    C = out["panop_predictions"][1]["voxel_logits"].C.clone()
    C[3, 2] = 20                                                                        # y = min_C + 24: past the box
    out["panop_predictions"][1]["voxel_logits"] = CR.Rows(out["panop_predictions"][1]["voxel_logits"].F, C)
    with pytest.raises(ValueError, match="1 mask rows outside the box"):
        PR.step_entries(out, batch, [1])
    out, batch = _case(g, 1)
    with pytest.raises(ValueError, match="CUDA tensors"):                              # a valid subnet on the host
        PR.step_entries(out, batch, [0])


def test_step_checks_the_evaluated_subnets():
    net = parity.pasconet(M=2, f=16, num_queries=8, in_channels=16)
    with pytest.raises(ValueError, match=r"subnets \[0, 1\]"):
        net.step({}, None, None, metrics={0: MT.Evaluator(1, uncertainty=False)})


# ---- GPU ------------------------------------------------------------------------------------------------------------
def _evaluators(subnets):
    return {i: MT.Evaluator(n_entries=1, n_classes=K, uncertainty=False) for i in subnets}


@pytest.mark.gpu
def test_fixture_counts_match_the_reference():
    g = parity.fixture(GOLD)
    evs = _evaluators(range(M))
    for step in range(STEPS):
        out, batch = _case(g, step, "cuda")
        PR.evaluate_step(out, batch, evs)
        for m in range(M):
            tag, acc = f"after{step}_m{m}", evs[m]._e[0]
            cats = g[tag + "_pq_cats"].tolist()
            assert sorted(acc.cats) == cats, (tag, sorted(acc.cats), cats)
            for c, want in zip(cats, g[tag + "_pq_fields"]):
                all_iou, all_n, iou, tp, fp, fn = acc.cats[c].fields()
                assert (tp, fp, fn, all_n) == (int(want[3]), int(want[4]), int(want[5]), want[1]), (tag, c)
                for got, ref in ((iou, want[2]), (all_iou, want[0])):
                    assert abs(got - ref) <= 4e-7 * max(1.0, abs(ref)), (tag, c, got, ref)
            assert [acc.c_tp, acc.c_fp, acc.c_fn] == g[tag + "_completion"].tolist(), tag
            np.testing.assert_array_equal(np.stack([acc.tps, acc.fps, acc.fns]), g[tag + "_class_counts"], err_msg=tag)
    assert (g["after0_m1_pq_fields"][:, 3:5] == 0).all()                       # subnet 1 of step 0 keeps no query


@pytest.mark.gpu
def test_rows_outside_the_box_raise_on_the_device():
    g = parity.fixture(GOLD)
    out, batch = _case(g, 0, "cuda")
    ev = _evaluators([0])
    C = out["panop_predictions"][0]["voxel_logits"].C.clone()
    C[[0, 7], 1] = 7                                                                  # x = min_C − 1
    out["panop_predictions"][0]["voxel_logits"] = CR.Rows(out["panop_predictions"][0]["voxel_logits"].F, C)
    with pytest.raises(ValueError, match="2 mask rows outside the box"):
        PR.evaluate_step(out, batch, ev)
    assert ev[0]._e[0].c_tp == 0 and not ev[0]._e[0].cats and ev[0].last_scene == []


def _net_case(M, f=16, Q=20):
    from pasco_b200.synthetic import make_scene, training_batch
    torch.manual_seed(0)
    net = parity.pasconet(M=M, f=f, num_queries=Q, in_channels=16).cuda().train()
    sc = training_batch(make_scene((64, 64, 8), 0.1, M, 16, K, seed=0, n_masks=6))
    crit = CR.SetCriterion(K, [torch.ones(K + 1, device="cuda")] * M, torch.ones(K, device="cuda"))
    return net, sc, crit


def _recording_forward(net, monkeypatch):
    outs = []
    real = net.forward

    def fwd(*a, **k):
        outs.append(real(*a, **k))
        return outs[-1]
    monkeypatch.setattr(net, "forward", fwd)
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_step_without_metrics_is_fused_training_loss(M, monkeypatch):
    net, sc, crit = _net_case(M)
    outs = _recording_forward(net, monkeypatch)
    total, terms = net.step(sc, crit, net.class_frequencies)
    want, want_terms = CR.fused_training_loss(outs[0], sc, crit, net.class_frequencies)
    assert "loss_ce" in terms and list(terms) == list(want_terms)
    assert torch.equal(total, want)
    for k in terms:
        assert torch.equal(torch.as_tensor(terms[k]), torch.as_tensor(want_terms[k])), k
    # with metrics the loss is the same: the evaluation runs under no_grad on the same forward
    evs = _evaluators(evaluated_subnets(M))
    total2, _ = net.step(sc, crit, net.class_frequencies, metrics=evs)
    want2, _ = CR.fused_training_loss(outs[1], sc, crit, net.class_frequencies)
    assert torch.equal(total2, want2)
    assert all(len(ev.last_scene) == 1 for ev in evs.values())


@pytest.mark.gpu
def test_pretraining_epoch_trains_the_completion_loss_only(monkeypatch):
    net, sc, crit = _net_case(3)
    calls = []
    for cls, name in ((CR.SetCriterion, "__call__"), (CR.SetCriterion, "level_losses"), (CR.HungarianMatcher, "__call__"),
                      (CR.HungarianMatcher, "cost"), (CR.DeviceCriterion, "add_subnet")):
        real = getattr(cls, name)
        monkeypatch.setattr(cls, name, lambda self, *a, _r=real, _n=name, **k: calls.append(_n) or _r(self, *a, **k))
    outs = _recording_forward(net, monkeypatch)
    evs = _evaluators([0, 2])
    total, terms = net.step(sc, crit, net.class_frequencies, epoch=0, metrics=evs)
    assert list(terms) == ["compl_ce_loss", "compl_lovasz_loss"]
    assert "panop_predictions" not in outs[0]
    assert torch.isfinite(total) and total.requires_grad
    assert calls == []
    for ev in evs.values():
        assert ev.last_scene == [] and ev._e[0].c_tp == 0 and not ev._e[0].cats
    total, terms = net.step(sc, crit, net.class_frequencies, epoch=1, metrics=evs)     # the gate opens at epoch 1
    assert "loss_ce" in terms and "panop_predictions" in outs[1]
    assert all(len(ev.last_scene) == 1 for ev in evs.values())


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_evaluation_host_syncs(M):
    import warnings
    net, sc, crit = _net_case(M, f=16, Q=20)
    with torch.no_grad():
        out = net([f.cuda() for f in sc["in_feats"]], [c.cuda() for c in sc["in_coords"]], sc["global_min_Cs"],
                  sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"])
    subnets = evaluated_subnets(M)
    PR.evaluate_step(out, sc, _evaluators(subnets))                    # warm the allocator: a first cudaMalloc may sync
    torch.cuda.synchronize()
    evs = _evaluators(subnets)
    counts = []
    for fn in (lambda: PR.step_entries(out, sc, subnets), lambda: PR.evaluate_step(out, sc, evs)):
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                fn()
            finally:
                torch.cuda.set_sync_debug_mode("default")
        counts.append([f"{os.path.basename(x.filename)}:{x.lineno}" for x in w if "called a synchronizing" in str(x.message)])
    assert len(counts[0]) == len(subnets) * PR.STEP_ENTRY_SYNCS, counts
    assert len(counts[1]) == len(subnets) * (PR.STEP_ENTRY_SYNCS + MT.VAL_UPDATE_SYNCS), counts


_REF = pytest.mark.skipif(not os.path.isdir(os.path.join(parity.REF, "pasco")),
                          reason="no upstream PaSCo checkout was readable when build() ran: oracle/_ref not staged")


@pytest.mark.gpu
@_REF
def test_step_metrics_match_the_unmodified_reference_step():
    """PascoNet.step's evaluators against Net.step(batch, "train")'s pq_stat["train"][i] / ssc_metrics["train"][i] on the
    drop-in, hooks off, recipe weights, the 64x64x8 fixture scene at M = 2 (min_C = 0, no cap active)."""
    from pasco_b200 import ops
    from pasco_b200.synthetic import training_batch
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    dev = torch.device("cuda")
    meta = parity.manifest("net_cfg1_m2_manifest.json")
    ME, ref = parity.reference_net(n_infers=2)
    sd = fill_state_dict(ref.state_dict())
    ref.load_state_dict(sd)
    ref.to(dev).train()
    mine = parity.pasconet(M=2)
    mine.load_reference_state_dict(sd)
    mine.to(dev).train()
    sc = training_batch(parity.scene(meta, M=2))
    assert all(int(c.abs().sum()) == 0 for c in sc["min_Cs"])
    d = lambda t: t.to(dev)  # noqa: E731
    ref_batch = dict(sc, min_Cs=[d(c) for c in sc["min_Cs"]], max_Cs=[d(c) for c in sc["max_Cs"]], Ts=[d(t) for t in sc["Ts"]],
                     global_min_Cs=d(sc["global_min_Cs"]), global_max_Cs=d(sc["global_max_Cs"]),
                     geo_labels={"1_1": d(sc["geo_labels"]["1_1"])})
    ref.class_weights = [torch.ones(K + 1, device=dev) for _ in range(2)]
    ref.criterion.class_weights = ref.class_weights
    ref.criterion.compl_labelweights = torch.ones(K, device=dev)
    ref.object_mask_threshold = 0.05
    ref.step(ref_batch, "train")
    crit = CR.SetCriterion(K, [torch.ones(K + 1, device=dev)] * 2, torch.ones(K, device=dev))
    evs = _evaluators([0, 1])
    outs = []
    real = mine.forward
    mine.forward = lambda *a, **k: outs.append(real(*a, **k)) or outs[-1]
    mine.step(sc, crit, mine.class_frequencies, metrics=evs, object_mask_threshold=0.05)
    thing_ids = list(PR.THING_IDS)
    for i in (0, 1):
        pq, ssc, acc = ref.pq_stat["train"][i], ref.ssc_metrics["train"][i], evs[i]._e[0]
        assert sorted(acc.cats) == sorted(pq.pq_per_cat), i
        for c in pq.pq_per_cat:
            r, e = pq.pq_per_cat[c], acc.cats[c]
            assert (e.tp, e.fp, e.fn, e.all_n) == (r.tp, r.fp, r.fn, r.all_n), (i, c)
        assert [acc.c_tp, acc.c_fp, acc.c_fn] == [ssc.completion_tp, ssc.completion_fp, ssc.completion_fn], i
        # the two networks' semantic logits agree to ~1e-5 (DESIGN.md §4), so a cell whose two best classes are closer
        # than 1e-3 may take the other class in the reference: each such cell moves at most four per-class counts by 1
        top2 = outs[0]["sem_logits_at_scales"][1][i].F.detach().topk(2, dim=1).values
        near = int((top2[:, 0] - top2[:, 1] < 1e-3).sum())
        diff = np.abs(np.stack([acc.tps, acc.fps, acc.fns]) - np.stack([ssc.tps, ssc.fps, ssc.fns]))
        assert int(diff.sum()) <= 4 * near, (i, int(diff.sum()), near)
        got = evs[i].compute()[0]
        for name, isthing in (("All", None), ("Things", True), ("Stuff", False)):
            want = pq.pq_average(isthing, 0, thing_ids)[0]
            for k in ("pq", "sq", "rq"):
                assert abs(got[name][k] - float(want[k])) <= 1e-6, (i, name, k, got[name][k], float(want[k]))
