"""pasco_b200/criterion.py against the reference's OWN loss code (pasco/loss/criterion_sparse.py, matcher_sparse.py,
losses.py, lovasz.py), whose outputs on a synthetic M = 2 prediction set are stored in tests/golden/loss_m2.npz by
tests/golden/make_golden_loss.py (which also checks its composition of the total against the reference's real `Net.step`).
CPU tests: the criterion is device-agnostic torch code (+ the SciPy assignment on the host, as in the reference)."""
import os

import numpy as np
import pytest
import torch

from pasco_b200 import criterion as CR

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "loss_m2.npz")
M, LEVELS = 2, 4


@pytest.fixture(scope="module")
def gold():
    return dict(np.load(GOLD))


def _t(a, grad=False):
    t = torch.as_tensor(np.asarray(a))
    return t.clone().requires_grad_(True) if grad else t


def _inputs(g, grad=False):
    leaves = {}

    def leaf(name):
        leaves[name] = _t(g[name], grad)
        return leaves[name]
    sem_at = {s: [CR.Rows(leaf(f"sem{s}_F_m{m}"), _t(g[f"sem{s}_C_m{m}"])) for m in range(M)] for s in (1, 2, 4)}
    preds = []
    for m in range(M):
        lv = [{"voxel_logits": CR.Rows(leaf(f"vox_F_m{m}_l{l}"), _t(g[f"vox_C_m{m}"])), "query_logits": leaf(f"query_m{m}_l{l}")}
              for l in range(LEVELS)]
        lv[0]["aux_outputs"] = lv[1:]
        preds.append(lv[0])
    sem = _t(g["semantic_label"])
    batch = {"sem_labels": {f"1_{s}": _t(g[f"sem_labels_1_{s}"]) for s in (1, 2, 4)},
             "min_Cs": [_t(g["min_C"])] * M, "max_Cs": [_t(g["max_C"])] * M, "semantic_label": sem,
             "mask_label": [{"labels": _t(g["labels"][m]), "masks": _t(g["masks"][m])} for m in range(M)],
             "geo_labels": {"1_1": torch.where(sem == 255, 255.0, (sem > 0).float())}}
    freqs = {f"1_{s}": g["class_frequencies"][i] for i, s in enumerate((1, 2, 4))}
    crit = CR.SetCriterion(20, list(_t(g["class_weights"])), _t(g["compl_labelweights"]))
    return {"sem_logits_at_scales": sem_at, "panop_predictions": preds}, batch, freqs, crit, leaves


def _close(a, b, tol=2e-6):
    return abs(float(a) - float(b)) <= tol * max(1.0, abs(float(b)))


def test_completion_loss_matches_reference_both_datasets(gold):
    out, batch, freqs, _, _ = _inputs(gold)
    ce, lov = CR.completion_loss(batch["sem_labels"], out["sem_logits_at_scales"], batch["min_Cs"], batch["max_Cs"], freqs)
    assert _close(ce, gold["compl_ce"]) and _close(lov, gold["compl_lovasz"]), (float(ce), float(lov))
    ce, lov = CR.completion_loss(batch["sem_labels"], out["sem_logits_at_scales"], batch["min_Cs"], batch["max_Cs"], freqs,
                                 power=1 / 1.5)                       # losses.py:69-118 (KITTI-360 label weights)
    assert _close(ce, gold["compl_ce_kitti360"]) and _close(lov, gold["compl_lovasz_kitti360"])


def test_every_criterion_term_and_assignment_matches_reference(gold):
    out, batch, _, crit, _ = _inputs(gold)
    for m, pred in enumerate(out["panop_predictions"]):
        ml = batch["mask_label"][m]
        ls = crit(pred, ml["labels"], ml["masks"], batch["semantic_label"][m], batch["geo_labels"]["1_1"][m] == 255, m,
                  batch["min_Cs"][m], main_ssc=True)
        for lv, (qi, tj) in enumerate(crit.last_indices):
            assert np.array_equal(torch.stack([qi, tj]).numpy(), gold[f"match_m{m}_l{lv}"]), f"assignment m{m} level {lv}"
        for k in ("loss_ce", "loss_mask", "loss_dice", "ssc_ce_loss", "ssc_lovasz_loss"):
            assert _close(ls[k], gold[f"{k}_m{m}"]), (k, m, float(ls[k]), float(gold[f"{k}_m{m}"]))
        assert len(ls["loss_aux"]) == 5 * (LEVELS - 1)
        for k, v in ls["loss_aux"].items():
            assert _close(v, gold[f"{k}_m{m}"]), (k, m, float(v), float(gold[f"{k}_m{m}"]))


def test_total_and_gradients_match_net_step_composition(gold):
    out, batch, freqs, crit, leaves = _inputs(gold, grad=True)
    total, terms = CR.training_loss(out, batch, crit, freqs)
    assert _close(total, gold["total"]), (float(total), float(gold["total"]))
    assert "ssc_ce_loss" not in terms and "ssc_ce_loss_level0" in terms        # the main level's ssc terms are not in the total
    total.backward()
    for name, t in leaves.items():
        ref = torch.as_tensor(gold[f"grad_{name}"])
        got = t.grad if t.grad is not None else torch.zeros_like(t)
        scale = float(ref.abs().max())
        assert float((got - ref).abs().max()) <= 2e-5 * max(scale, 1e-12) + 1e-9, (name, float((got - ref).abs().max()), scale)
        if name.startswith(("vox_F", "query")):
            assert scale > 0, name


def test_lovasz_batched_equals_the_per_class_loop():
    g = torch.Generator().manual_seed(1)
    logits, labels = torch.randn(500, 7, generator=g), torch.randint(0, 7, (500,), generator=g)
    labels[labels == 5] = 2                                                    # class 5 absent
    probs = logits.softmax(1)
    per = []
    for c in range(7):
        fg = (labels == c).float()
        if fg.sum() == 0 or c == 0:
            continue
        err, perm = torch.sort((fg - probs[:, c]).abs(), descending=True)
        fs = fg[perm]
        jac = 1 - (fs.sum() - fs.cumsum(0)) / (fs.sum() + (1 - fs).cumsum(0))
        jac[1:] = jac[1:] - jac[:-1].clone()
        per.append(torch.dot(err, jac))
    assert torch.allclose(CR.lovasz_softmax_flat(logits, labels, ignores=(0,)), torch.stack(per).mean(), atol=1e-6)
    assert float(CR.lovasz_softmax_flat(logits[:0], labels[:0])) == 0.0


def test_degenerate_inputs():
    """All queries dustbin → no ssc term (helper.py:38-39 returns None); no voxel inside the bounds → that pair is skipped."""
    q = torch.zeros(5, 21)
    q[:, 20] = 9.0
    assert CR.semantic_inference(torch.rand(10, 5), q) is None
    rows = CR.Rows(torch.randn(4, 20), torch.tensor([[0, 99, 99, 99]] * 4, dtype=torch.int32))
    ce, lov = CR.completion_loss({"1_1": torch.zeros(1, 8, 8, 8, dtype=torch.uint8)}, {1: [rows]}, [torch.zeros(3)],
                                 [torch.full((3,), 7)], {"1_1": np.ones(20)})
    assert float(ce) == 0.0 and float(lov) == 0.0


@pytest.mark.gpu
def test_criterion_on_the_device_matches_reference(gold):
    """Same fixture on cuda:0."""
    dev = torch.device("cuda:0")
    out, batch, freqs, crit, leaves = _inputs(gold, grad=True)

    def mv(x):
        if isinstance(x, torch.Tensor):
            return x.detach().to(dev).requires_grad_(x.requires_grad)
        if isinstance(x, CR.Rows):
            return CR.Rows(mv(x.F), mv(x.C))
        if isinstance(x, dict):
            return {k: mv(v) for k, v in x.items()}
        if isinstance(x, list):
            return [mv(v) for v in x]
        return x
    out_d, batch_d = mv(out), mv(batch)
    tf32 = torch.backends.cuda.matmul.allow_tf32       # whatever an earlier test left behind: the comparison is fp32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        total, terms = CR.training_loss(out_d, batch_d, crit, freqs)
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    assert _close(total, gold["total"], 1e-4), (float(total), float(gold["total"]))
    total.backward()
    g = out_d["panop_predictions"][0]["voxel_logits"].F.grad.cpu()
    ref = torch.as_tensor(gold["grad_vox_F_m0_l0"])
    assert float((g - ref).abs().max()) <= 1e-3 * float(ref.abs().max())
