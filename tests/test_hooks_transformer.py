"""The transformer hook (pasco_b200/hooks.py install(transformer=True)): the unmodified reference's
PositionEmbeddingSineSparse.forward on ops.sine_pos (csrc/posenc.cu), TransformerPredictorV2.pred_heads on
net3d.mask_head and, with the attention group, the projections and per-item outputs of its forward; and PascoNet's
MaskTransformer on the same shared functions.

  * CPU: the new C-ABI symbol is declared and typed, no local memory in the new kernel, install / uninstall
    restore every patched name, alone and together with the attention group;
  * GPU: the encoding against the reference module bit for bit (int32 / int64, [P, 4] / [P, 3], zero, negative and
    ±32767 coordinates, P = 1 / 4095 / 2 M, n = 128 / 32), add mode into a column slice, the mask head, the whole
    hooked forward against the golden fixtures, independent coordinates per level, Net.step + backward with the group
    off and on, every fallback, host synchronisations, and PascoNet's MaskTransformer against its torch restatement.
GPU tests that need the reference skip when oracle/_ref is not staged.
"""
import collections
import copy
import math
import os
import re
import subprocess
import sys
import warnings

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
K = 20
PATCHED = (("pasco.models.transformer.position_encoding", "PositionEmbeddingSineSparse", "forward"),
           ("pasco.models.transformer.transformer_predictor_v2", "TransformerPredictorV2", "pred_heads"),
           ("pasco.models.transformer.transformer_predictor_v2", "TransformerPredictorV2", "forward"),
           ("pasco.models.transformer.blocks", "CrossAttentionLayer", "forward"))


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_new_symbol_declared_and_typed():
    from pasco_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pasco_sm100.h")).read(), flags=re.S)
    m = re.search(r"\bpasco_sine_pos\s*\(([^;)]*)\)\s*;", src)
    assert m, "pasco_sine_pos not declared"
    n_args = len([a for a in m.group(1).split(",") if a.strip()])
    assert len(_lib.PROTOTYPES["pasco_sine_pos"][1]) == n_args


def test_new_kernel_uses_no_local_memory():
    from pasco_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = 0
    for f in re.split(r"\n\s*Function : ", sass):
        head = f.split("\n")[0]
        if "posenc_cu" in head and "k_sine_pos" in head:
            found += 1
            assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert found == 2                                   # int32 and int64 coordinates


def _classes():
    import importlib
    parity.reference_net()
    return [(getattr(importlib.import_module(m), c), n) for m, c, n in PATCHED]


@needs_ref
@pytest.mark.parametrize("with_attention", [False, True])
def test_install_uninstall_restores_every_name(with_attention):
    from pasco_b200 import hooks
    classes = _classes()
    names = lambda: tuple(getattr(c, n) for c, n in classes)  # noqa: E731
    hooks.uninstall()
    before = names()
    for _ in range(2):
        assert hooks.install(attention=with_attention, transformer=True)
    got = names()
    assert got[:2] == (hooks._pe_forward, hooks._pred_heads)
    assert got[2:] == ((hooks._transformer_forward, hooks._cross_attention_forward) if with_attention else before[2:])
    for (c, n), fn in zip(classes[:2], before[:2]):
        assert getattr(c, "_pasco_b200_orig_" + n) is fn
    for _ in range(2):
        hooks.uninstall()
    assert names() == before


# ------------------------------------------------------------------------------------------------
# GPU: the sine encoding
# ------------------------------------------------------------------------------------------------
def _ref_pe(n, **kw):
    parity.reference_net()
    from pasco.models.transformer.position_encoding import PositionEmbeddingSineSparse
    pe = PositionEmbeddingSineSparse(n, normalize=True, **kw)
    orig = getattr(PositionEmbeddingSineSparse, "_pasco_b200_orig_forward", PositionEmbeddingSineSparse.forward)
    return pe, lambda c: orig(pe, c)                    # the reference's own forward, installed hooks or not


def _coords(P, cols, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    c = torch.randint(-40, 300, (P, cols), generator=g)
    special = torch.tensor([0, -1, 1, -31, 31, -32, 32, -33, 33, -64, 64, -65, 65, 32767, -32767, 255])
    k = min(P, 64)
    c[:k, -3:] = special[torch.randint(0, len(special), (k, 3), generator=g)]
    if cols == 4:
        c[:, 0] = torch.randint(0, 3, (P,), generator=g)
    return c.to(dtype).cuda()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("P", [1, 4095, 2_000_000])
@pytest.mark.parametrize("n", [128, 32])
@pytest.mark.parametrize("dtype", [torch.int32, torch.int64])
@pytest.mark.parametrize("cols", [4, 3])
def test_sine_pos_equals_the_reference_module(P, n, dtype, cols):
    from pasco_b200 import ops
    _, ref = _ref_pe(n)
    c = _coords(P, cols, dtype, seed=P + n + cols)
    want = ref(c[:, cols - 3:])
    got = ops.sine_pos(c, n)
    assert got.shape == (P, 3 * n) and torch.equal(got, want)
    if P == 4095:                                       # a [P, 3] view of the [P, 4] rows, with its row pitch
        assert torch.equal(ops.sine_pos(c[:, cols - 3:], n), want)


@pytest.mark.gpu
@needs_ref
def test_sine_pos_covers_every_int16_coordinate():
    """Each axis on its own: every coordinate of [-32768, 32767] against the reference module."""
    from pasco_b200 import ops
    _, ref = _ref_pe(128)
    v = torch.arange(-32768, 32768, device="cuda", dtype=torch.int32)
    c = torch.stack([v, v.flip(0), torch.zeros_like(v)], 1)
    assert torch.equal(ops.sine_pos(c, 128), ref(c))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("n", [128, 32])
def test_add_mode_equals_y_plus_pe(n):
    from pasco_b200 import ops
    _, ref = _ref_pe(n)
    P = 5000
    c = _coords(P, 4, torch.int32, seed=3)
    pe = ref(c[:, 1:])
    y = torch.randn(P, 3 * n, device="cuda")
    want = y + pe
    assert torch.equal(ops.sine_pos(c, n, out=y, add=True), want) and torch.equal(y, want)
    wide = torch.randn(P, 3 * n + 70, device="cuda")           # a column slice with a row pitch
    before = wide.clone()
    view = wide[:, 5:5 + 3 * n]
    want = view + pe
    ops.sine_pos(c, n, out=view, add=True)
    assert torch.equal(wide[:, 5:5 + 3 * n], want)
    assert torch.equal(wide[:, :5], before[:, :5]) and torch.equal(wide[:, 5 + 3 * n:], before[:, 5 + 3 * n:])
    ops.sine_pos(c, n, out=view)                                # write mode into the slice
    assert torch.equal(wide[:, 5:5 + 3 * n], pe)
    # autograd: d(y + pe)/dy is the identity
    x = torch.randn(P, 64, device="cuda", requires_grad=True)
    w = torch.randn(3 * n, 64, device="cuda")
    g = torch.randn(P, 3 * n, device="cuda")
    out = ops.add_sine_pos(x @ w.t(), c, n)
    assert torch.equal(out.detach(), (x @ w.t()).detach() + pe)
    out.backward(g)
    gx = x.grad.clone()
    x.grad = None
    ((x @ w.t()) + pe).backward(g)
    assert torch.equal(gx, x.grad)


# ------------------------------------------------------------------------------------------------
# GPU: the mask head
# ------------------------------------------------------------------------------------------------
def _predictor(B, Q, hidden=384):
    parity.reference_net()
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    torch.manual_seed(0)
    return TransformerPredictorV2([64, 64, 64], hidden_dim=hidden, num_queries=Q, n_infers=B, mask_dim=64,
                                  num_classes=K, dim_feedforward=256).cuda()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("Q", [100, 200])
def test_mask_head_matches_pred_heads(B, Q):
    from pasco_b200 import hooks, ops
    from pasco_b200.net3d import mask_head
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    ops.set_precision("fp32")
    hooks.uninstall()
    tp = _predictor(B, Q)
    g = torch.Generator(device="cuda").manual_seed(1)
    out = torch.randn(B, Q, 384, device="cuda", generator=g)
    feat = torch.randn(B, 30_000, 384, device="cuda", generator=g)
    cls_w, msk_w = TransformerPredictorV2.pred_heads(tp, out, feat)
    cls_g, msk_g = mask_head(tp, out, feat)
    assert torch.equal(cls_g, cls_w)
    assert msk_g.shape == msk_w.shape == (B, 30_000, Q)
    err = parity.relerr(msk_g, msk_w)
    print(f"B={B} Q={Q}: mask logits relative error {err:.2e}")
    assert err <= 1e-3
    assert hooks.install(attention=False, transformer=True)
    try:
        cls_h, msk_h = tp.pred_heads(out, feat)
    finally:
        hooks.uninstall()
    assert torch.equal(cls_h, cls_g) and torch.equal(msk_h, msk_g)


# ------------------------------------------------------------------------------------------------
# GPU: the whole hooked forward
# ------------------------------------------------------------------------------------------------
def _reference(M):
    from pasco_b200 import ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    ME, net = parity.reference_net(n_infers=M)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    return ME, net.cuda().train()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_hooked_forward_matches_golden(M):
    from pasco_b200 import hooks
    man = parity.manifest("net_cfg1_manifest.json" if M == 1 else "net_cfg1_m2_manifest.json")
    ME, net = _reference(M)
    sc = parity.scene(man, M)
    hooks.uninstall()
    try:
        assert hooks.install(attention=True)
        torch.manual_seed(0)
        off = parity.forward_reference(ME, net, sc, "cuda")
        assert hooks.install(attention=True, transformer=True)
        torch.manual_seed(0)
        out = parity.forward_reference(ME, net, sc, "cuda")
        gold = parity.fixture("net_cfg1.npz" if M == 1 else "net_cfg1_m2.npz")
        report = parity.check_outputs(out, gold, man, sem=False, worst=M == 2)
        print(f"reference M={M}, attention + transformer hooks vs golden:", report)
        for m in range(M):
            a, b = out["panop_predictions"][m], off["panop_predictions"][m]
            assert set(a) == set(b) == {"query_logits", "voxel_logits", "aux_outputs"}
            assert len(a["aux_outputs"]) == len(b["aux_outputs"]) == 3
            for x, y in zip([a] + a["aux_outputs"], [b] + b["aux_outputs"]):
                assert set(x) == set(y)
                assert torch.equal(x["voxel_logits"].C, y["voxel_logits"].C)        # keep_pad's rows, in order
                assert x["voxel_logits"].F.shape == y["voxel_logits"].F.shape
                assert x["query_logits"].shape == y["query_logits"].shape
                assert parity.relerr(x["query_logits"], y["query_logits"]) <= 1e-3
        # every level's coordinates are a tensor of their own
        p = out["panop_predictions"][0]
        levels = [p["voxel_logits"]] + [a["voxel_logits"] for a in p["aux_outputs"]]
        saved = [lv.C.clone() for lv in levels]
        levels[0].C[:, 1:] -= 7
        assert torch.equal(levels[0].C[:, 1:], saved[0][:, 1:] - 7)
        for lv, s in zip(levels[1:], saved[1:]):
            assert torch.equal(lv.C, s)
    finally:
        hooks.uninstall()


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified Net's training step, the other six groups on, transformer off and on
# ------------------------------------------------------------------------------------------------
def _set(hooks, transformer):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=True, decoder=True,
                         transformer=transformer)


def _val(v):
    return float(v.detach()) if torch.is_tensor(v) else float(v)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_net_training_step_transformer_off_and_on(M, capsys):
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    hooks.uninstall()
    _, net = parity.reference_net(n_infers=M)
    net.class_weights = [torch.ones(K + 1) for _ in range(M)]
    net.criterion.class_weights = net.class_weights
    net.criterion.compl_labelweights = torch.ones(K)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    net.to(dev).train()
    meta = parity.INFER_MANIFEST["cases"]["m2" if M == 2 else "m1"]
    sc = parity.scene(meta, M)
    grid = tuple(meta["grid"])
    g = torch.Generator().manual_seed(5)
    sem = torch.randint(0, K, (M,) + grid, generator=g)
    sem[torch.rand(sem.shape, generator=g) < 0.6] = 0
    sem[:, :, :2, :] = 255
    mask_label = []
    for m in range(M):
        present = [c for c in range(1, K) if (sem[m] == c).any()]
        mask_label.append({"labels": torch.tensor(present, dtype=torch.uint8, device=dev),
                           "masks": torch.stack([sem[m] == c for c in present]).to(dev)})
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 sem_labels=sc["sem_labels"], semantic_label=sem.to(torch.uint8).to(dev),
                 geo_labels={"1_1": torch.where(sem == 255, 255.0, (sem > 0).float()).to(dev)}, mask_label=mask_label)
    state = copy.deepcopy(net.state_dict())

    def step(transformer):
        _set(hooks, transformer)
        net.load_state_dict(state)
        logged = {}
        net.log = lambda k, v, **kw: logged.__setitem__(k, _val(v))
        net.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        out = net.step(batch, "train")
        out["loss"].backward()
        grads = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
        return _val(out["loss"]), logged, grads

    try:
        want = step(False)
        got = step(True)
    finally:
        hooks.uninstall()
    capsys.readouterr()
    assert set(got[1]) == set(want[1])
    for k, v in want[1].items():
        assert abs(got[1][k] - v) <= 1e-3 * max(1.0, abs(v)), (k, got[1][k], v)
    assert set(got[2]) == set(want[2])
    num = sum(float((got[2][n] - want[2][n]).double().norm() ** 2) for n in want[2]) ** 0.5
    den = sum(float(want[2][n].double().norm() ** 2) for n in want[2]) ** 0.5
    print(f"M = {M}: loss {got[0]:.6f} (transformer on) vs {want[0]:.6f} (off); gradients relative L2 {num / den:.2e}")
    assert num / den < 1e-2


# ------------------------------------------------------------------------------------------------
# GPU: fallbacks
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "unnormalized", "scale", "odd_n", "wide_n", "float"])
def test_pe_fallbacks(case):
    from pasco_b200 import hooks
    parity.reference_net()
    from pasco.models.transformer.position_encoding import PositionEmbeddingSineSparse as PE
    n, kw = {"odd_n": (127, {}), "wide_n": (258, {}), "unnormalized": (128, {"normalize": False}),
             "scale": (128, {"normalize": True, "scale": 1.0})}.get(case, (128, {"normalize": True}))
    pe = PE(n, **kw)
    c = _coords(300, 3, torch.int32, seed=9)
    if case == "cpu":
        c = c.cpu()
    if case == "float":
        c = c.float() + 0.5
    calls = []
    hooks.uninstall()
    assert hooks.install(attention=False, transformer=True)
    orig = PE._pasco_b200_orig_forward
    PE._pasco_b200_orig_forward = lambda self, x: calls.append(1) or orig(self, x)
    try:
        if case == "odd_n":                             # the reference's own stack of n/2 + 1 and n/2 columns raises
            with pytest.raises(RuntimeError):
                pe(c)
        else:
            got = pe(c)
    finally:
        PE._pasco_b200_orig_forward = orig
        hooks.uninstall()
    assert calls == [1]
    if case != "odd_n":
        assert torch.equal(got, pe(c))


@pytest.mark.gpu
@needs_ref
def test_glue_fallbacks():
    """pred_heads on CPU tensors goes to the original; a hidden size other than 3n, or the transformer group without
    the attention group, leaves the forward's glue on the reference's own code."""
    from pasco_b200 import hooks
    from pasco.models.transformer.position_encoding import PositionEmbeddingSineSparse as PE
    tp = _predictor(1, 100)
    xs = {s: (None, torch.zeros(1, 8, 4, dtype=torch.int32, device="cuda")) for s in (4, 2, 1)}
    hooks.uninstall()
    assert hooks.install(attention=False, transformer=True)
    try:
        assert not hooks._transformer_glue(tp, xs)                      # no attention group
        assert hooks.install(attention=True, transformer=True)
        assert hooks._transformer_glue(tp, xs)
        tp.pe_layer = PE(64, normalize=True)                             # 3n = 192 != hidden 384
        assert not hooks._transformer_glue(tp, xs)
        tp.pe_layer = PE(128, normalize=False)
        assert not hooks._transformer_glue(tp, xs)
        tp.pe_layer = PE(128, normalize=True)
        calls = []
        orig = type(tp)._pasco_b200_orig_pred_heads
        type(tp)._pasco_b200_orig_pred_heads = lambda self, o, f: calls.append(1) or orig(self, o, f)
        try:
            tp.cpu().pred_heads(torch.randn(1, 100, 384), torch.randn(1, 50, 384))
        finally:
            type(tp)._pasco_b200_orig_pred_heads = orig
        assert calls == [1]
    finally:
        hooks.uninstall()


# ------------------------------------------------------------------------------------------------
# GPU: host synchronisations and repeats
# ------------------------------------------------------------------------------------------------
def _syncs(fn):
    torch.cuda.synchronize()
    with warnings.catch_warnings(record=True) as w:
        warnings.simplefilter("always")
        torch.cuda.set_sync_debug_mode("warn")
        try:
            out = fn()
        finally:
            torch.cuda.set_sync_debug_mode("default")
    return out, [f"{os.path.basename(v.filename)}:{v.lineno}" for v in w if "called a synchronizing" in str(v.message)]


@pytest.mark.gpu
@needs_ref
def test_syncs_bounded_and_repeats_identical():
    from pasco_b200 import hooks, ops
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    man = parity.manifest("net_cfg1_m2_manifest.json")
    ME, net = _reference(2)
    sc = parity.scene(man, 2)
    got = {}

    def record(this, xs, sem, lo, hi, keep_pad):
        got["args"] = (xs, sem, lo, hi, keep_pad)
        return inner(this, xs, sem, lo, hi, keep_pad)

    hooks.uninstall()
    assert hooks.install(attention=True, transformer=True)
    inner = TransformerPredictorV2.forward
    TransformerPredictorV2.forward = record
    try:
        torch.manual_seed(0)
        parity.forward_reference(ME, net, sc, "cuda")
    finally:
        TransformerPredictorV2.forward = inner
    tp = net.transformer_predictor
    try:
        outs, counts = [], collections.defaultdict(set)
        for _ in range(3):
            with torch.no_grad():
                preds, s_all = _syncs(lambda: TransformerPredictorV2.forward(tp, *got["args"]))
            glue = [s for s in s_all if s.startswith("hooks.py:")]
            counts["forward"].add(len(s_all))
            counts["glue"].add(len(glue))
            outs.append([t for p in preds for lv in [p] + p["aux_outputs"]
                         for t in (lv["query_logits"], lv["voxel_logits"].F, lv["voxel_logits"].C)])
            xs = got["args"][0]
            _, s_pe = _syncs(lambda: tp.pe_layer(xs[1][1].reshape(-1, 4)[:, 1:]))
            _, s_proj = _syncs(lambda: hooks._proj_plus_pos(tp.input_projs[0], xs[4][0], xs[4][1], 128))
            counts["pe+proj"].add(len(s_pe) + len(s_proj))
        for a, b in zip(outs[0], outs[-1]):
            assert torch.equal(a, b)
    finally:
        hooks.uninstall()
    print("host synchronisations per hooked forward:", dict(counts))
    assert all(len(v) == 1 for v in counts.values()), counts
    assert next(iter(counts["glue"])) <= hooks.TRANSFORMER_SYNCS
    assert counts["pe+proj"] == {0}
    assert ops.CALLS > 0


# ------------------------------------------------------------------------------------------------
# GPU: PascoNet's MaskTransformer against its torch restatement
# ------------------------------------------------------------------------------------------------
def _torch_sine(coords, n, temperature=10000.0):
    """position_encoding.py:90-135 with normalize=True in torch, as PascoNet computed it before ops.sine_pos."""
    c = coords.float()
    c = c / (c + 1e-6) * (2 * math.pi)
    dim_t = torch.arange(n, dtype=torch.float32, device=c.device)
    dim_t = temperature ** (2 * torch.div(dim_t, 2, rounding_mode="floor") / n)
    outs = []
    for a in range(3):
        p = c[:, a, None] / dim_t
        outs.append(torch.cat([p[:, 0::2].sin(), p[:, 1::2].cos()], 1))
    return torch.cat(outs, 1)


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_pasconet_mask_transformer_equals_torch_encoding(M, monkeypatch):
    from pasco_b200 import net3d, ops
    ops.set_precision("fp32")
    man = parity.manifest("net_cfg1_manifest.json" if M == 1 else "net_cfg1_m2_manifest.json")
    net = parity.pasconet(M, recipe=True).cuda().train()
    calls = []
    fwd = net3d.MaskTransformer.forward

    def record(self, feats, subnet=0):
        calls.append((self, feats, subnet))
        return fwd(self, feats, subnet)

    monkeypatch.setattr(net3d.MaskTransformer, "forward", record)
    with torch.no_grad():
        parity.forward(net, parity.scene(man, M))
    monkeypatch.setattr(net3d.MaskTransformer, "forward", fwd)
    assert calls
    for tf, feats, subnet in calls:
        with torch.no_grad():
            got = fwd(tf, feats, subnet)
            with monkeypatch.context() as mp:
                mp.setattr(net3d, "proj_plus_pos", lambda lin, F_, C, n: ops.linear(F_, lin.weight, lin.bias)
                           + _torch_sine(C[:, 1:], n))
                want = fwd(tf, feats, subnet)
        for a, b in zip(got[0] + got[1], want[0] + want[1]):
            assert torch.equal(a, b)
        assert torch.equal(net3d.sine_position_encoding(feats[1][1][:, 1:], 128), _torch_sine(feats[1][1][:, 1:], 128))
