"""The post-processing hooks (pasco_b200/hooks.py install(postprocess=True)): the unmodified reference's
Ensembler.ensemble_sem_compl / ensemble_panop and panoptic_inference on the panoptic kernels, against the reference's own
saved originals (`_pasco_b200_orig_*`) on the same inputs.

  * CPU: install / uninstall restore every patched attribute (both Net modules' panoptic_inference included), install()
    without arguments patches the attention alone;
  * GPU: panoptic_inference on make_golden_predict.scene_a rows at Q = 24, 100 and 200 (merged stuff, no kept query, one
    kept query, a zero-area query, voxel logits, a training-frame call with negative min_C, a scale-8 scene size and
    unsorted rows), the Ensembler at M = 1, 2, 3 under identity, flip + translation and 7-degree poses, fallbacks, bit-
    identical repeats, host synchronisations independent of Q, and the unmodified Net end to end: step_inference with
    eval=True on a seeded ground truth (outputs and accumulated metrics) and one training step (loss bit for bit, metrics).
GPU tests skip when oracle/_ref is not staged.
"""
import collections
import os
import sys
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_predict as GP  # noqa: E402
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
SIZE = (256, 256, 32)
THING_IDS = GP.THING_IDS


def _reference():
    parity.reference_net()                     # sys.path + import asserts: `pasco` from oracle/_ref on pasco_b200.me
    import MinkowskiEngine as ME
    from pasco.models import ensembler, helper, net_panoptic_sparse
    return ME, ensembler, helper, net_panoptic_sparse


@pytest.fixture
def hooked():
    from pasco_b200 import hooks, ops
    ops.set_precision("fp32")
    mods = _reference()
    assert hooks.install(attention=False, postprocess=True)
    try:
        yield mods
    finally:
        hooks.uninstall()


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
@needs_ref
def test_install_uninstall_restores_every_attribute():
    from pasco_b200 import hooks
    _, ensembler, helper, nps = _reference()
    from pasco.models.transformer import blocks
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    E = ensembler.Ensembler
    before = (E.ensemble_sem_compl, E.ensemble_panop, helper.panoptic_inference, nps.panoptic_inference,
              blocks.CrossAttentionLayer.forward, TransformerPredictorV2.compute_attn_mask)
    users = [m for m in hooks._users()]
    assert nps in users and helper in users
    assert hooks.install()                                      # no arguments: the attention alone
    assert blocks.CrossAttentionLayer.forward is hooks._cross_attention_forward
    assert E.ensemble_panop is before[1] and nps.panoptic_inference is before[3]
    for _ in range(2):
        assert hooks.install(postprocess=True)
    assert E.ensemble_sem_compl is hooks._ensemble_sem_compl and E.ensemble_panop is hooks._ensemble_panop
    assert all(m.panoptic_inference is hooks._panoptic_inference for m in users)
    assert nps._pasco_b200_orig_panoptic_inference is before[2]
    for _ in range(2):
        hooks.uninstall()
    after = (E.ensemble_sem_compl, E.ensemble_panop, helper.panoptic_inference, nps.panoptic_inference,
             blocks.CrossAttentionLayer.forward, TransformerPredictorV2.compute_attn_mask)
    assert all(a is b for a, b in zip(after, before))
    assert all(m.panoptic_inference is before[2] for m in users)


# ------------------------------------------------------------------------------------------------
# panoptic_inference, hooked vs original
# ------------------------------------------------------------------------------------------------
def _rows(ME, Q, seed=0, logits=False, shift=(0, 0, 0), perm=False):
    """Subnet 0 of scene_a at Q queries as the reference's inputs: (voxel SparseTensor, query probabilities [1, Q, 21])."""
    preds, _, _ = GP.scene_a(seed=seed, M=1, Q=Q)
    lg, c = preds[0]["voxel_logits"]
    c = c.int() + torch.tensor(shift, dtype=torch.int32)
    if perm:
        p = torch.randperm(c.shape[0], generator=torch.Generator().manual_seed(seed))
        lg, c = lg[p], c[p]
    C4 = torch.cat([torch.zeros_like(c[:, :1]), c], 1).cuda()
    F = lg.cuda() if logits else torch.sigmoid(lg.cuda())
    return ME.SparseTensor(F, C4), torch.softmax(preds[0]["query_logits"].cuda(), -1)


def _compare(a, b):
    """hooked a vs original b: labels, segments, ins_uncertainty, all-mask probabilities exactly; vox_confidence and
    vox_uncertainty within 1e-6 relative; shapes and dtypes everywhere."""
    assert set(a) == set(b)
    for k in ("panoptic_seg_denses", "semantic_seg_denses", "ins_uncertainty_denses", "vox_confidence_denses",
              "vox_uncertainty_denses"):
        assert a[k].shape == b[k].shape and a[k].dtype == b[k].dtype and a[k].device == b[k].device, k
    for x, y in zip(a["vox_all_mask_probs_denses"], b["vox_all_mask_probs_denses"]):
        assert x.shape == y.shape and x.dtype == y.dtype
        assert torch.equal(x, y)
    differ = int((a["panoptic_seg_denses"] != b["panoptic_seg_denses"]).sum())
    assert differ == 0, f"{differ} voxels with another panoptic label"
    assert torch.equal(a["semantic_seg_denses"], b["semantic_seg_denses"])
    assert torch.equal(a["ins_uncertainty_denses"], b["ins_uncertainty_denses"])
    for k in ("vox_confidence_denses", "vox_uncertainty_denses"):
        torch.testing.assert_close(a[k], b[k], rtol=1e-6, atol=0)
    assert len(a["panoptic_seg_sparses"]) == 1 and torch.equal(a["panoptic_seg_sparses"][0], b["panoptic_seg_sparses"][0])
    sa, sb = a["segments_infos"][0], b["segments_infos"][0]
    assert len(sa) == len(sb)
    for x, y in zip(sa, sb):
        assert set(x) == set(y)
        for k in ("id", "isthing", "category_id", "query_id", "confidence"):
            assert x[k] == y[k] and type(x[k]) is type(y[k]), k
        assert torch.equal(x["all_class_probs"], y["all_class_probs"])


def _both(helper, *args, **kw):
    from pasco_b200 import hooks
    got = hooks._panoptic_inference(*args, **kw)
    ref = helper._pasco_b200_orig_panoptic_inference(*args, **kw)
    _compare(got, ref)
    return got


TEST_KW = dict(overlap_threshold=0.4, thing_ids=THING_IDS, scene_size=SIZE, min_C=torch.tensor([0, 0, 0], dtype=torch.int32),
               input_query_logit=False, input_voxel_logit=False)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("Q", [24, 100, 200])
def test_panoptic_inference_matches_the_original(hooked, Q):
    ME, _, helper, _ = hooked
    vox, qp = _rows(ME, Q)
    got = _both(helper, vox, qp, object_mask_threshold=0.7, **TEST_KW)
    pan, sem = got["panoptic_seg_denses"][0], got["semantic_seg_denses"][0]
    assert len(got["segments_infos"][0]) >= 4
    assert ((pan != 0) & (sem == 0)).any(), "a stuff class merged"
    merged = (pan != 0) & (sem == 0)
    assert not got["ins_uncertainty_denses"][0][merged].any() and not got["vox_uncertainty_denses"][0][merged].any()
    assert got["vox_uncertainty_denses"].gt(0).any()


@pytest.mark.gpu
@needs_ref
def test_panoptic_inference_edge_cases(hooked):
    ME, _, helper, _ = hooked
    vox, qp = _rows(ME, 100)
    # no kept query: kq = 0 gives a [0, X, Y, Z] all-mask volume
    got = _both(helper, vox, qp, object_mask_threshold=0.9999, **TEST_KW)
    assert got["vox_all_mask_probs_denses"][0].shape == (0,) + SIZE and got["segments_infos"][0] == []
    # one kept query: [X, Y, Z]
    q1 = qp.clone()
    top = int(q1[0].max(-1)[0].argmax())
    q1[0, :, 1:] = 0.0
    q1[0, :, 0] = 1.0
    q1[0, top] = qp[0, top]
    got = _both(helper, vox, q1, object_mask_threshold=0.2, **TEST_KW)
    assert got["vox_all_mask_probs_denses"][0].shape == SIZE and len(got["segments_infos"][0]) == 1
    # a kept query of zero area (every mask probability below the occupancy threshold)
    F = vox.F.clone()
    F[:, top] = 0.1
    _both(helper, ME.SparseTensor(F, vox.C), qp, object_mask_threshold=0.2, **TEST_KW)
    # voxel and query logits
    vl, _ = _rows(ME, 100, logits=True)
    _both(helper, vl, torch.log(qp), object_mask_threshold=0.7, **dict(TEST_KW, input_voxel_logit=True,
                                                                       input_query_logit=True))


@pytest.mark.gpu
@needs_ref
def test_panoptic_inference_training_frame(hooked):
    """Net.step's call: the subnet's own frame (negative min_C on the host), compute_scene_size(..., scale=8) and rows in
    manager order (unsorted)."""
    ME, _, helper, _ = hooked
    from pasco.models.misc import compute_scene_size
    vox, qp = _rows(ME, 100, shift=(-70, -60, -5), perm=True)
    C = vox.C[:, 1:].cpu()
    min_C, max_C = C.min(0)[0], C.max(0)[0]
    size = compute_scene_size(min_C, max_C, scale=8).int()
    assert (min_C < 0).any() and bool((size % 8 == 0).all())
    kw = dict(TEST_KW, scene_size=size, min_C=min_C)
    got = _both(helper, vox, qp, object_mask_threshold=0.7, **kw)
    assert tuple(got["panoptic_seg_denses"].shape[1:]) == tuple(size.tolist())
    _both(helper, vox, qp, object_mask_threshold=0.7, **dict(kw, min_C=min_C.cuda()))


@pytest.mark.gpu
@needs_ref
def test_panoptic_inference_fallbacks(hooked, monkeypatch):
    ME, _, helper, _ = hooked
    from pasco_b200 import hooks, ops
    calls = []
    # the original only records the call: on rows outside the box its own indexing would read out of bounds
    monkeypatch.setattr(hooks, "_orig_panoptic_inference", lambda *a: calls.append(1))
    vox, qp = _rows(ME, 24)

    def reaches_original(q, **kw):
        n = len(calls)
        hooks._panoptic_inference(vox, q, object_mask_threshold=0.7, **dict(TEST_KW, **kw))
        return len(calls) == n + 1

    # a row outside the box: the flag is raised, cleared, and the original decides
    assert reaches_original(qp, scene_size=(200, 256, 32))
    assert int(ops._err_flag(vox.F.device).item()) == 0
    assert reaches_original(qp, min_C=torch.tensor([100, 0, 0]))
    assert reaches_original(qp.repeat(2, 1, 1))                                              # batch size 2
    assert reaches_original(torch.softmax(torch.randn(1, 24, 70, device="cuda"), -1))       # 69 classes + dustbin
    assert reaches_original(qp.cpu())                                                        # CPU query probabilities
    assert len(calls) == 5


@pytest.mark.gpu
@needs_ref
def test_panoptic_inference_repeat_syncs_and_launches(hooked):
    ME, _, helper, _ = hooked
    from pasco_b200 import hooks
    counts = {}
    for Q in (100, 200):
        vox, qp = _rows(ME, Q)
        a = hooks._panoptic_inference(vox, qp, object_mask_threshold=0.7, **TEST_KW)
        b = hooks._panoptic_inference(vox, qp, object_mask_threshold=0.7, **TEST_KW)
        for k in a:
            if torch.is_tensor(a[k]):
                assert torch.equal(a[k], b[k]), k
        assert torch.equal(a["vox_all_mask_probs_denses"][0], b["vox_all_mask_probs_denses"][0])
        torch.cuda.synchronize()
        with warnings.catch_warnings(record=True) as w:
            warnings.simplefilter("always")
            torch.cuda.set_sync_debug_mode("warn")
            try:
                hooks._panoptic_inference(vox, qp, object_mask_threshold=0.7, **TEST_KW)
            finally:
                torch.cuda.set_sync_debug_mode("default")
        sites = collections.Counter(f"{os.path.basename(x.filename)}:{x.lineno}" for x in w
                                    if "synchroniz" in str(x.message) and f"{os.sep}pasco_b200{os.sep}" in x.filename)
        counts[Q] = sum(sites.values())
        print(f"Q = {Q}: host synchronisations by call site {dict(sites)}")
    assert counts[100] == counts[200] > 0


# ------------------------------------------------------------------------------------------------
# Ensembler, hooked vs original
# ------------------------------------------------------------------------------------------------
def _ensembler_inputs(ME, M, Q=100, seed=0):
    preds, sems, Ts = GP.scene_a(seed=seed, M=M, Q=Q)
    bc = lambda c: torch.cat([torch.zeros_like(c[:, :1]), c], 1).int().cuda()  # noqa: E731
    sem_at = {1: [ME.SparseTensor(f.cuda(), bc(c)) for f, c in sems]}
    ref_preds = [{"voxel_logits": ME.SparseTensor(p["voxel_logits"][0].cuda(), bc(p["voxel_logits"][1])),
                  "query_logits": p["query_logits"].cuda()} for p in preds]
    return sem_at, ref_preds, [T.cuda() for T in Ts[:M]]


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2, 3])
def test_ensembler_matches_the_original(hooked, M):
    ME, ensembler, _, _ = hooked
    from pasco_b200 import hooks
    E = ensembler.Ensembler
    ens = E()
    sem_at, preds, Ts = _ensembler_inputs(ME, M)
    got_sem = ens.ensemble_sem_compl(sem_at, Ts)
    ref_sem = E._pasco_b200_orig_ensemble_sem_compl(ens, sem_at, Ts)
    assert len(got_sem) == len(ref_sem) == M + 1
    for g, r in zip(got_sem, ref_sem):
        assert g.shape == r.shape and g.dtype == r.dtype
        torch.testing.assert_close(g, r, rtol=0, atol=1e-6)
    gate = ens._pasco_b200_sem_state[1].view(SIZE)
    assert torch.equal(gate.bool(), got_sem[-1].argmax(0) != 0)
    got = ens.ensemble_panop(preds, got_sem, (32, 32, 4), Ts, iou_threshold=0.2, measure_time=True)
    ref = E._pasco_b200_orig_ensemble_panop(ens, preds, ref_sem, (32, 32, 4), Ts, iou_threshold=0.2, measure_time=True)
    assert len(got) == len(ref) == M + 1
    for i, (g, r) in enumerate(zip(got, ref)):
        assert set(g) == set(r) and g["ensemble_time"] >= 0
        assert torch.equal(g["voxel_probs"].C.cpu(), r["voxel_probs"].C.int().cpu()), f"rows of entry {i}"
        torch.testing.assert_close(g["voxel_probs"].F, r["voxel_probs"].F, rtol=0, atol=1e-5)
        assert g["query_probs"].shape == r["query_probs"].shape
        torch.testing.assert_close(g["query_probs"], r["query_probs"], rtol=0, atol=1e-6)
        torch.testing.assert_close(g["sem_probs"].F, r["sem_probs"].F, rtol=0, atol=1e-6)
    # state that does not belong to the volumes passed: the gate is recomputed from them
    ens._pasco_b200_sem_state = (torch.zeros(1), torch.zeros(1))
    again = hooks._ensemble_panop(ens, preds, got_sem, SIZE, Ts, iou_threshold=0.2)
    for g, a in zip(got, again):
        assert torch.equal(g["voxel_probs"].C, a["voxel_probs"].C) and torch.equal(g["voxel_probs"].F, a["voxel_probs"].F)


@pytest.mark.gpu
@needs_ref
def test_ensembler_fallbacks(hooked, monkeypatch):
    ME, ensembler, _, _ = hooked
    E = ensembler.Ensembler
    calls = []
    for name in ("_pasco_b200_orig_ensemble_sem_compl", "_pasco_b200_orig_ensemble_panop"):
        monkeypatch.setattr(E, name, lambda *a, **k: calls.append(1))          # records the routing only
    sem_at, preds, Ts = _ensembler_inputs(ME, 1, Q=24)
    ens = E()
    vols = ens.ensemble_sem_compl(sem_at, Ts)
    assert calls == []

    def reaches_original(fn, *a):
        n = len(calls)
        fn(*a)
        return len(calls) == n + 1

    two = [dict(p, query_logits=p["query_logits"].repeat(2, 1, 1)) for p in preds]
    assert reaches_original(ens.ensemble_panop, two, vols, SIZE, Ts)                       # batch size 2
    assert reaches_original(ens.ensemble_sem_compl, {1: sem_at[1] * 9}, Ts * 9)            # M = 9
    assert reaches_original(ens.ensemble_panop, preds * 9, vols, SIZE, Ts * 9)
    s = sem_at[1][0]
    wide = {1: [ME.SparseTensor(torch.randn(s.F.shape[0], 70, device="cuda"), s.C)]}
    assert reaches_original(ens.ensemble_sem_compl, wide, Ts)                              # 70 classes
    assert reaches_original(ens.ensemble_panop, preds, [v.cpu() for v in vols], SIZE, Ts)  # CPU volumes


# ------------------------------------------------------------------------------------------------
# end to end: the unmodified Net with and without the hooks
# ------------------------------------------------------------------------------------------------
def _gt(grid, size, seed, K=20):
    """A seeded ground truth over the scene's box (make_golden_eval.gt_scene's recipe on this scene): class boxes as masks,
    the semantic label the last box's class, an unknown slab.  Returns (semantic uint8 [*size], mask label)."""
    g = torch.Generator().manual_seed(seed)
    sem = torch.zeros(size, dtype=torch.uint8)
    items = []
    for j in range(10):
        cls = [1, 2, 9, 3, 9, 10, 4, 5, 11, 6][j]
        lo = [int(torch.randint(0, max(1, grid[d] - 8), (1,), generator=g)) for d in range(3)]
        hi = [min(grid[d], lo[d] + int(torch.randint(3, 12, (1,), generator=g))) for d in range(3)]
        box = tuple(slice(a, b) for a, b in zip(lo, hi))
        m = torch.zeros(size, dtype=torch.bool)
        m[box] = True
        sem[box] = cls
        items.append((cls, m))
    sem[grid[0] // 2:grid[0] // 2 + 2] = 255
    return sem, {"labels": torch.tensor([c for c, _ in items]), "masks": torch.stack([m for _, m in items])}


def _same_state(a, b, path="", tol=1e-6, depth=0):
    """Two metric objects / containers: integers and booleans exactly, floats within tol (relative to 1)."""
    if depth > 6:
        return
    if isinstance(a, dict):
        assert set(a) == set(b), path
        for k in a:
            _same_state(a[k], b[k], f"{path}.{k}", tol, depth + 1)
    elif isinstance(a, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same_state(x, y, f"{path}[{i}]", tol, depth + 1)
    elif torch.is_tensor(a) or isinstance(a, np.ndarray) or isinstance(a, (int, float, np.number, bool)):
        x = torch.as_tensor(a).detach().cpu().double()
        y = torch.as_tensor(b).detach().cpu().double()
        assert x.shape == y.shape, path
        if x.dtype.is_floating_point and not (isinstance(a, (int, bool, np.integer)) or
                                              (torch.is_tensor(a) and not a.is_floating_point())):
            assert torch.allclose(x, y, rtol=tol, atol=tol, equal_nan=True), (path, x, y)
        else:
            assert torch.equal(x, y), (path, x, y)
    elif isinstance(a, torch.nn.Module) or callable(a):
        return
    elif hasattr(a, "__dict__"):
        _same_state(vars(a), vars(b), path, tol, depth + 1)
    else:
        assert a == b, path


def _fresh_metrics(net, step):
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics
    for i in net.pq_stat[step]:
        net.pq_stat[step][i] = PQStat()
        net.ssc_metrics[step][i] = SSCMetrics(net.n_classes)
        net.uncertainty_metrics[step][i] = UncertaintyMetrics()


def _metrics(net, step):
    return {"pq": {i: {c: vars(v) for c, v in p.pq_per_cat.items()} for i, p in net.pq_stat[step].items()},
            "ssc": {i: vars(m) for i, m in net.ssc_metrics[step].items()},
            "unc": {i: vars(m) for i, m in net.uncertainty_metrics[step].items()}}


@pytest.mark.gpu
@needs_ref
def test_net_step_inference_with_and_without_hooks():
    """scripts/eval.py's Net.step_inference(batch, "test", eval=True) on a seeded ground truth: the outputs and every
    metric the reference accumulates (PQStat, SSC counts, uncertainty ECE / NLL) agree with and without the hooks."""
    from pasco_b200 import hooks, ops
    ops.set_precision("fp32")
    ME, net = parity.reference_net()
    net, _ = parity.load_eval(net, "m1", ref_names=False)
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    meta = parity.INFER_MANIFEST["cases"]["m1"]
    sc = parity.scene(meta)
    plain = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"])
    sem, mask_label = _gt(meta["grid"], SIZE, 7)
    # one more ground-truth instance on most of a predicted segment, so that a match at IoU > 0.5 is reached
    with torch.no_grad():
        pred = net.step_inference(plain, "test")[0][0]
    seg = pred["segments_infos"][0][0]
    inst = (pred["panoptic_seg_denses"][0] == seg["id"]).cpu()
    inst[:2] = False
    sem[inst] = seg["category_id"]
    mask_label = {"labels": torch.cat([mask_label["labels"], torch.tensor([seg["category_id"]])]).to(dev),
                  "masks": torch.cat([mask_label["masks"], inst[None]]).to(dev)}
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"],
                 semantic_label=sem.unsqueeze(0).to(dev), semantic_label_origin=sem.unsqueeze(0).to(dev),
                 mask_label=[mask_label], mask_label_origin=[mask_label])
    with torch.no_grad():
        _fresh_metrics(net, "test")
        ref = net.step_inference(batch, "test", eval=True)[0]
        ref_metrics = _metrics(net, "test")
        _fresh_metrics(net, "test")
        assert hooks.install(attention=False, postprocess=True)
        try:
            c0 = ops.CALLS
            with parity.launches() as launches:
                got = net.step_inference(batch, "test", eval=True, measure_time=True)[0]
            assert ops.CALLS - c0 > 100 and not [x for x in launches if x[1] == "simt"]
            assert len(net.ensemble_times) == 1 and net.ensemble_times[0] > 0
        finally:
            hooks.uninstall()
        got_metrics = _metrics(net, "test")
    assert len(got) == len(ref) == 2
    for g, r in zip(got, ref):
        _compare({k: v for k, v in g.items() if k != "ssc_confidence"}, {k: v for k, v in r.items() if k != "ssc_confidence"})
        torch.testing.assert_close(g["ssc_confidence"], r["ssc_confidence"], rtol=0, atol=1e-6)
    segs = [len(g["segments_infos"][0]) for g in got]
    tp = [sum(v["tp"] for v in got_metrics["pq"][i].values()) for i in got_metrics["pq"]]
    print("segments per entry:", segs, "PQ true positives per entry:", tp)
    assert sum(segs) > 0 and sum(tp) > 0
    _same_state(got_metrics, ref_metrics)


@pytest.mark.gpu
@needs_ref
def test_net_training_step_with_and_without_hooks():
    """scripts/train.py's Net.step(batch, "train"): panoptic_inference on subnets 0 and M − 1 with grad-carrying
    probabilities, device min_C and compute_scene_size's device size.  Same loss bit for bit, same "train" metrics."""
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    ME, net = parity.reference_net(n_infers=2)
    K = net.n_classes
    net.class_weights = [torch.ones(K + 1) for _ in range(2)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    net.to(dev).train()
    meta = parity.INFER_MANIFEST["cases"]["m2"]
    sc = parity.scene(meta, 2)
    grid = tuple(meta["grid"])
    g = torch.Generator().manual_seed(5)
    sem = torch.randint(0, K, (2,) + grid, generator=g)
    sem[torch.rand(sem.shape, generator=g) < 0.6] = 0
    sem[:, :, :2, :] = 255
    mask_label = []
    for m in range(2):
        present = [c for c in range(1, K) if (sem[m] == c).any()]
        mask_label.append({"labels": torch.tensor(present, dtype=torch.uint8, device=dev),
                           "masks": torch.stack([sem[m] == c for c in present]).to(dev)})
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 sem_labels=sc["sem_labels"], semantic_label=sem.to(torch.uint8).to(dev),
                 geo_labels={"1_1": torch.where(sem == 255, 255.0, (sem > 0).float()).to(dev)}, mask_label=mask_label)

    def step():
        _fresh_metrics(net, "train")
        torch.manual_seed(0)
        out = net.step(batch, "train")
        return out, _metrics(net, "train")

    ref, ref_metrics = step()
    assert hooks.install(attention=False, postprocess=True)
    try:
        got, got_metrics = step()
    finally:
        hooks.uninstall()
    assert torch.equal(got["loss"], ref["loss"]), (float(got["loss"]), float(ref["loss"]))
    assert len(got["panop_out_subnets"]) == len(ref["panop_out_subnets"]) == 2
    for a, b in zip(got["panop_out_subnets"], ref["panop_out_subnets"]):
        _compare(a, b)
    print("train segments per evaluated subnet:", [len(a["segments_infos"][0]) for a in got["panop_out_subnets"]])
    _same_state(got_metrics, ref_metrics)
