"""Inference mode (scripts/eval.py: model.eval(), forward(test=True) without gradients): every BatchNorm normalises with
its running statistics, and the engine folds them into the convolutions —

  * the convolution's inference epilogue (pasco_conv_forward_planes_infer, ops.conv_infer) against the composition of
    existing ops (conv + affine_act + split_planes), bit for bit, at every column-range width, in fp32 and bf16 mode;
  * PascoNet.eval() and the unmodified reference on the drop-in against golden vectors the unmodified reference produced
    in eval mode on the CPU oracle (tests/golden/make_golden_infer.py, running statistics calibrated there and stored);
  * PascoNet's fused eval forward bit for bit against the same forward with the fusions off (ops.inference_fusion);
  * the unmodified Net.step_inference (eval.py's path: ensembling + panoptic post-processing) on the drop-in;
  * CPU: which calls take the fused forms, the fixture manifest, the new entry point's header and ctypes signature.
"""
import json
import os
import re
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
GOLD = os.path.join(HERE, "golden")
sys.path.insert(0, GOLD)
from recipe import fill_state_dict  # noqa: E402

MANIFEST = json.load(open(os.path.join(GOLD, "net_cfg1_infer_manifest.json")))
STAT_SUFFIXES = (".running_mean", ".running_var")


def _pasconet(M=1):
    from pasco_b200.net3d import PascoNet
    torch.manual_seed(0)
    return PascoNet(n_classes=20, n_infers=M, in_channels=283, f=64, num_queries=100, heavy_decoder=False)


# ------------------------------------------------------------------------------------------------
# CPU: routing, manifest, signature
# ------------------------------------------------------------------------------------------------
class _NoSplitLib:
    @staticmethod
    def pasco_conv_splitk_workspace_bytes(K, n_out, c_out):
        return 0


def test_routing_predicates(monkeypatch):
    """bn_act_conv: training → the fused BNActConv, eval + gradients → the differentiable row path (unchanged), eval
    without gradients → the split fusion; ResBlock.infer_ok / the drop-in's deferred BatchNorm follow the same predicate."""
    from pasco_b200 import ops
    monkeypatch.setattr(ops, "load", lambda: _NoSplitLib)
    bn = torch.nn.BatchNorm1d(64)
    x = types.SimpleNamespace(is_cuda=True)
    w = torch.empty(27, 64, 64)
    kmap = types.SimpleNamespace(K=27, nbr=object(), n_out=100_000, n_in=100_000)
    net = _pasconet()

    def route():
        return ops.bn_act_conv_route(bn, x, w, kmap)

    for grad in (True, False):
        with torch.set_grad_enabled(grad):
            bn.train()
            net.train()
            assert route() == "fused" and not ops.inference_fusion_active(bn) and not ops.inference_fusion_active(net)
            bn.eval()
            net.eval()
            assert route() == ("unfused" if grad else "eval_split")
            assert ops.inference_fusion_active(bn) == (not grad) and ops.inference_fusion_active(net) == (not grad)
    with torch.no_grad():
        ops.inference_fusion(False)
        try:
            assert route() == "unfused" and not ops.inference_fusion_active(net)
        finally:
            ops.inference_fusion(True)
        assert route() == "eval_split"
        assert ops.bn_act_conv_route(bn, types.SimpleNamespace(is_cuda=False), w, kmap) == "unfused"
        assert ops.bn_act_conv_route(torch.nn.BatchNorm1d(64, track_running_stats=False).eval(), x, w, kmap) == "unfused"
        # a shape off the plane-gather path (register gather: identity rows) keeps the row path
        assert ops.bn_act_conv_route(bn, x, torch.empty(1, 64, 64), types.SimpleNamespace(K=1, nbr=None, n_out=10, n_in=10)) == "unfused"
        ops.force_simt(True)
        try:
            assert route() == "unfused"
        finally:
            ops.force_simt(False)


def test_eval_coefficients_are_batchnorm_eval():
    from pasco_b200 import ops
    torch.manual_seed(0)
    bn = torch.nn.BatchNorm1d(32)
    with torch.no_grad():
        bn.weight.uniform_(0.5, 1.5)
        bn.bias.normal_()
        bn.running_mean.normal_()
        bn.running_var.uniform_(0.5, 2.0)
    bn.eval()
    x = torch.randn(100, 32)
    scale, shift = ops.bn_eval_coefs(bn)
    torch.testing.assert_close(x * scale + shift, bn(x), rtol=1e-6, atol=1e-6)


def test_infer_fixture_manifest_matches_pasconet():
    """Every running statistic PascoNet holds (M = 1 and M = 2) is in the fixture of each case, with its shape, and each
    case holds the summaries of every output."""
    for tag, case in MANIFEST["cases"].items():
        M = case["n_infers"]
        z = np.load(os.path.join(GOLD, f"net_cfg1_infer_{tag}.npz"))
        mine = {k: list(v.shape) for k, v in _pasconet(M).reference_state_dict().items() if k.endswith(STAT_SUFFIXES)}
        ref = case["running_stats"]
        assert sorted(mine) == sorted(ref), (tag, sorted(set(ref) ^ set(mine))[:5])
        assert all(mine[k] == ref[k] for k in ref), tag
        for k, shape in ref.items():
            a = z[f"stat::{k}"]
            assert list(a.shape) == shape and np.isfinite(a).all()
            if k.endswith("running_var"):
                assert (a >= 0).all()
        for m in range(M):
            sfx = "" if M == 1 else f"_m{m}"
            for name in ("sem4", "sem2", "sem1", "vox"):
                n = int(z[f"{name}{sfx}_n"][0])
                assert n > 0 and len(z[f"{name}{sfx}_subK"]) == len(z[f"{name}{sfx}_subF"]) == (n + case["row_step"] - 1) // case["row_step"]
            for lvl in ["query_logits"] + [f"aux{i}_query_logits" for i in range(3)]:
                assert z[f"{lvl}{sfx}"].shape == (100, 21)
    assert sorted(MANIFEST["cases"]) == ["big", "m1", "m2"]
    assert int(np.load(os.path.join(GOLD, "net_cfg1_infer_big.npz"))["sem1_n"][0]) > 1_000_000


_CT = {"void*": "p", "int32_t*": "p", "float*": "p", "int64_t": "i64", "int32_t": "i32", "pasco_stream_t": "p"}


def test_infer_entry_point_header_matches_ctypes():
    from pasco_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pasco_sm100.h")).read(), flags=re.S)
    m = re.search(r"int\s+pasco_conv_forward_planes_infer\s*\(([^)]*)\)", src)
    assert m, "pasco_conv_forward_planes_infer is not declared"
    kinds = []
    for arg in m.group(1).split(","):
        t = " ".join(arg.replace("const", "").split()[:-1]).replace(" *", "*")
        if arg.strip().split()[-1].startswith("*"):
            t += "*"
        kinds.append(_CT[t])
    ctm = {_lib.C.c_void_p: "p", _lib.C.c_int64: "i64", _lib.C.c_int32: "i32"}
    res, args = _lib.PROTOTYPES["pasco_conv_forward_planes_infer"]
    assert res is _lib.C.c_int
    assert [ctm[a] for a in args] == kinds


# ------------------------------------------------------------------------------------------------
# GPU: the inference epilogue against the composition of existing ops
# ------------------------------------------------------------------------------------------------
def _launches():
    from pasco_b200 import ops
    torch.cuda.synchronize()
    out = [(kind, m["path"]) for kind, _, _, m in ops.PROFILE]
    ops.PROFILE = None
    ops.PAIR_COUNTS.clear()
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "bf16"])
@pytest.mark.parametrize("C", [16, 32, 64, 80, 128, 192, 256])
def test_inference_epilogue_is_the_unfused_sequence_bit_for_bit(C, precision):
    from pasco_b200 import ops
    ops.set_precision(precision)
    try:
        dev = torch.device("cuda")
        g = torch.Generator().manual_seed(C)
        n = 20_011                                   # 157 tiles: not a multiple of 128, not split over the offsets
        nbr = torch.randint(0, n, (27, n), generator=g, dtype=torch.int32)
        nbr[torch.rand(27, n, generator=g) < 0.6] = -1
        nbr[13] = torch.arange(n, dtype=torch.int32)
        kmap = ops.KernelMap(nbr.to(dev), n, n)
        W = (torch.randn(27, C, C, generator=g) / (27 * C) ** 0.5).to(dev)
        bias = torch.randn(1, C, generator=g).to(dev)
        x = torch.randn(n, C, generator=g).to(dev)
        res = torch.randn(n, C, generator=g).to(dev)
        sc0, sh0 = (torch.rand(C, generator=g) + 0.5).to(dev), torch.randn(C, generator=g).to(dev)
        sc1, sh1 = (torch.rand(C, generator=g) + 0.5).to(dev), torch.randn(C, generator=g).to(dev)
        assert ops.conv_path("fwd", C, C, 27, kmap.nbr, n) == "planes"
        packs = ops.PackedWeights()
        with torch.no_grad():
            planes = ops.split_planes(x, sc0, sh0, ops.ACT_RELU)
            for use_res, use_bias, use_next, want_out, act_out, act_next, coefs in (
                    (False, False, True, False, 0, ops.ACT_RELU, True),       # ResBlock conv1: planes of relu(BN2(y1)) only
                    (True, False, True, True, ops.ACT_RELU, ops.ACT_RELU, True),   # ResBlock conv2 followed by a block
                    (True, False, False, True, ops.ACT_RELU, 0, False),       # last ResBlock of a stage
                    (False, True, False, True, 0, 0, False),                  # plain convolution + bias
                    (True, True, True, False, ops.ACT_LEAKY, ops.ACT_LEAKY, True),
                    (False, True, True, True, 0, ops.ACT_LEAKY, False)):      # planes without an affine
                bias_t = bias if use_bias else None
                ops.PROFILE = []
                out, nxt = ops.conv_infer(planes, W, bias_t, kmap, packs, residual=res if use_res else None, act_out=act_out,
                                          want_out=want_out, next_coefs=(sc1, sh1) if coefs else None, next_act=act_next,
                                          want_next=use_next)
                assert _launches() == [("fwd", "planes_infer")]
                y = ops.conv_apply(x, W, kmap.nbr, n, False, None, bias_t.view(-1) if use_bias else None, packs=packs,
                                   planes=planes)
                if use_res:
                    y = ops.affine_act(y, None, None, act_out, res)
                tag = (C, precision, use_res, use_bias, use_next, want_out, act_out, act_next, coefs)
                assert (out is not None) == want_out and (nxt is not None) == use_next, tag
                if want_out:
                    assert torch.equal(out, y), tag
                if use_next:
                    ref = ops.split_planes(y, sc1, sh1, act_next) if coefs else ops.split_planes(y, None, None, act_next)
                    assert torch.equal(nxt[0], ref[0]), tag
                    assert (nxt[1] is None) == (precision == "bf16") and (nxt[1] is None or torch.equal(nxt[1], ref[1])), tag
        with pytest.raises(RuntimeError):
            ops.conv_infer(planes, W, None, kmap, packs)             # gradients enabled: refused
    finally:
        ops.PROFILE = None
        ops.set_precision("fp32")


# ------------------------------------------------------------------------------------------------
# GPU: networks in eval mode against the eval-mode golden vectors
# ------------------------------------------------------------------------------------------------
def _gold(tag):
    z = np.load(os.path.join(GOLD, f"net_cfg1_infer_{tag}.npz"))
    return {k: z[k] for k in z.files}


def _load_eval(net, tag, ref_names=True):
    """Recipe weights + the calibrated running statistics of fixture `tag`; eval mode."""
    gold = _gold(tag)
    sd = fill_state_dict(net.reference_state_dict() if ref_names else net.state_dict())
    n = 0
    for k in sd:
        if k.endswith(STAT_SUFFIXES) and f"stat::{k}" in gold:
            sd[k] = torch.from_numpy(gold[f"stat::{k}"]).to(sd[k].dtype)
            n += 1
    assert n == len(MANIFEST["cases"][tag]["running_stats"]), (n, tag)
    (net.load_reference_state_dict if ref_names else net.load_state_dict)(sd)
    return net.cuda().eval(), gold


def _check_golden(out, meta, gold, q=0.99):
    """test_golden_r2's checks (coordinate-set checksums, Σ, row subsample, query logits) plus the aux query logits."""
    from test_golden_r2 import _check_all
    rep = _check_all(out, meta, gold, q=q)
    for m in range(meta["n_infers"]):
        sfx = "" if meta["n_infers"] == 1 else f"_m{m}"
        for i, aux in enumerate(out["panop_predictions"][m]["aux_outputs"]):
            ref = torch.as_tensor(gold[f"aux{i}_query_logits{sfx}"]).double()
            e = float((aux["query_logits"][0].detach().cpu().double() - ref).abs().max() / ref.abs().max())
            rep[f"aux{i}{sfx}"] = e
            assert e <= 1e-3, (i, sfx, e)
    return rep


def _stats(net):
    return {k: v.clone() for k, v in net.state_dict().items() if k.endswith(STAT_SUFFIXES + (".num_batches_tracked",))}


def _run(net, b, fused=True):
    from pasco_b200 import ops
    dev = torch.device("cuda")
    ops.inference_fusion(fused)
    ops.PROFILE = []
    c0 = ops.CALLS
    try:
        with torch.no_grad():
            out = net([f.to(dev) for f in b["in_feats"]], [c.to(dev) for c in b["in_coords"]], b["global_min_Cs"],
                      b["global_max_Cs"], b["min_Cs"], b["max_Cs"], test=True)
        return out, ops.CALLS - c0, _launches()
    finally:
        ops.inference_fusion(True)
        ops.PROFILE = None


def _outputs(out, M):
    """(name, coordinates, features) of every output, for bit-for-bit comparison."""
    r = []
    for m in range(M):
        for s in (4, 2, 1):
            lg = out["sem_logits_at_scales"][s][m]
            r.append((f"sem{s}_{m}", lg.C, lg.F))
        p = out["panop_predictions"][m]
        r.append((f"vox_{m}", p["voxel_logits"].C, p["voxel_logits"].F))
        r.append((f"query_{m}", None, p["query_logits"]))
        r += [(f"aux{i}_{m}", None, a["query_logits"]) for i, a in enumerate(p["aux_outputs"])]
    return r


def _check_fused_vs_unfused(net, b, M):
    _run(net, b, fused=False)                                       # packs every weight: the counted runs pack none
    before = _stats(net)
    out, calls, launches = _run(net, b, fused=True)
    after = _stats(net)
    assert all(torch.equal(before[k], after[k]) for k in before), "the eval forward changed a running statistic"
    assert launches and not [x for x in launches if x[1] == "simt"], "a convolution ran on the CUDA cores"
    assert any(x[1] == "planes_infer" for x in launches), "no residual block ran on the inference epilogue"
    ref, calls_ref, launches_ref = _run(net, b, fused=False)
    assert not [x for x in launches_ref if x[1] == "planes_infer"]
    assert calls < calls_ref, (calls, calls_ref)
    for (name, c1, f1), (_, c2, f2) in zip(_outputs(out, M), _outputs(ref, M)):
        if c1 is not None:
            assert torch.equal(c1, c2), name
        assert torch.equal(f1, f2), name                           # value equality: -0 == +0
    return out, calls, calls_ref


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_pasconet_eval_matches_reference_eval_golden(M):
    from pasco_b200 import ops
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    meta = MANIFEST["cases"][f"m{M}"]
    net, gold = _load_eval(_pasconet(M), f"m{M}")
    b = make_scene(meta["grid"], meta["occ"], M, seed=meta["seed"])
    out, calls, calls_ref = _check_fused_vs_unfused(net, b, M)
    rep = _check_golden(out, meta, gold)
    print(f"eval M={M}: C-ABI calls fused {calls} / unfused {calls_ref};", rep)


@pytest.mark.gpu
def test_pasconet_eval_benchmark_scale_matches_reference_eval_golden():
    from pasco_b200 import ops
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    meta = MANIFEST["cases"]["big"]
    net, gold = _load_eval(_pasconet(1), "big")
    b = make_scene(meta["grid"], meta["occ"], 1, seed=meta["seed"])
    out, calls, calls_ref = _check_fused_vs_unfused(net, b, 1)
    # 1.74 M decoder voxels: argmax near-ties keep ~20 scale-1 and ~3 scale-2 voxels other than the CPU run (the parent
    # engine does the same; this forward is bit-identical to it), and a flipped voxel changes the features of its
    # neighbourhood through the residual blocks, the voxel head and the attention masks.  Measured on an H100: voxel-logit
    # row error 1.4e-4 at the 95th percentile, 8e-3 at the 99th; every other output 1.2e-4 at the 99th.  Bound: the 95th
    # percentile at 1e-3 and the median at 5e-4 (test_golden_r2's near-tie rule with the cap-branch quantile's margin).
    rep = _check_golden(out, meta, gold, q=0.95)
    print(f"eval benchmark scale: C-ABI calls fused {calls} / unfused {calls_ref};", rep)


def _reference_net():
    from test_dropin_reference import REF, _reference_net as make
    if not os.path.isdir(os.path.join(REF, "pasco")):
        pytest.skip("oracle/_ref not staged")
    return make()


@pytest.mark.gpu
def test_unmodified_reference_eval_on_the_engine_matches_golden():
    from pasco_b200 import ops
    from pasco_b200.synthetic import make_scene
    from test_dropin_reference import _forward_reference
    ops.set_precision("fp32")
    ME, net = _reference_net()
    net, gold = _load_eval(net, "m1", ref_names=False)
    dev = torch.device("cuda")
    meta = MANIFEST["cases"]["m1"]
    b = make_scene(meta["grid"], meta["occ"], 1, seed=meta["seed"])
    before = _stats(net)
    ops.PROFILE = []
    try:
        with torch.no_grad():
            out = _forward_reference(ME, net, b, dev, test=True)
        launches = _launches()
    finally:
        ops.PROFILE = None
    assert all(torch.equal(v, _stats(net)[k]) for k, v in before.items())
    assert launches and not [x for x in launches if x[1] == "simt"]
    rep = _check_golden(out, MANIFEST["cases"]["m1"], gold)
    print("drop-in eval vs golden:", rep)


class _RecordingBatch(dict):
    def __init__(self, *a, **k):
        super().__init__(*a, **k)
        self.read = set()

    def __getitem__(self, k):
        self.read.add(k)
        return super().__getitem__(k)


@pytest.mark.gpu
def test_unmodified_step_inference_runs_on_the_engine():
    """eval.py's path: Net.step_inference(batch, "test") in eval mode — the forward, the reference Ensembler and
    panoptic_inference (eval=False: no metrics)."""
    from pasco_b200 import ops
    from pasco_b200.synthetic import make_scene
    ops.set_precision("fp32")
    ME, net = _reference_net()
    net, _ = _load_eval(net, "m1", ref_names=False)
    dev = torch.device("cuda")
    meta = MANIFEST["cases"]["m1"]
    b = make_scene(meta["grid"], meta["occ"], 1, seed=meta["seed"])
    batch = _RecordingBatch(in_feats=[t.to(dev) for t in b["in_feats"]], in_coords=[t.to(dev) for t in b["in_coords"]],
                            min_Cs=[t.to(dev) for t in b["min_Cs"]], max_Cs=[t.to(dev) for t in b["max_Cs"]],
                            Ts=[t.to(dev) for t in b["Ts"]], global_min_Cs=b["global_min_Cs"].to(dev),
                            global_max_Cs=b["global_max_Cs"].to(dev),
                            geo_labels={k: v.to(dev) for k, v in b["sem_labels"].items()},
                            mask_classes=b["mask_classes"].to(dev))
    c0 = ops.CALLS
    with torch.no_grad():
        res = net.step_inference(batch, "test")
    torch.cuda.synchronize()
    assert ops.CALLS - c0 > 100
    assert batch.read <= {"in_feats", "in_coords", "min_Cs", "max_Cs", "Ts", "global_min_Cs", "global_max_Cs", "geo_labels"}, batch.read
    finite, n = [], 0

    def walk(o):
        nonlocal n
        if torch.is_tensor(o):
            n += 1
            if o.is_floating_point():
                finite.append(bool(torch.isfinite(o).all()))
        elif isinstance(o, dict):
            for v in o.values():
                walk(v)
        elif isinstance(o, (list, tuple)):
            for v in o:
                walk(v)
    walk(res)
    assert n > 0 and all(finite), (n, finite.count(False))
