"""Inference mode (scripts/eval.py: model.eval(), forward(test=True) without gradients): every BatchNorm normalises with
its running statistics, and the engine folds them into the convolutions —

  * the convolution's inference epilogue (pasco_conv_forward_planes_infer, ops.conv_infer) against the composition of
    existing ops (conv + affine_act + split_planes), bit for bit, at every column-range width, in fp32 and bf16 mode;
  * PascoNet.eval() and the unmodified reference on the drop-in against golden vectors the unmodified reference produced
    in eval mode on the CPU oracle (tests/golden/make_golden_infer.py, running statistics calibrated there and stored);
  * PascoNet's fused eval forward bit for bit against the same forward with the fusions off (ops.inference_fusion);
  * the unmodified Net.step_inference (eval.py's path: ensembling + panoptic post-processing) on the drop-in;
  * CPU: which calls take the fused forms, the fixture manifest.
"""
import os
import sys
import types

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from parity import STAT_SUFFIXES, INFER_MANIFEST as MANIFEST  # noqa: E402


# ------------------------------------------------------------------------------------------------
# CPU: routing, manifest, signature
# ------------------------------------------------------------------------------------------------
class _NoSplitLib:
    @staticmethod
    def pasco_conv_splitk_workspace_bytes(K, n_out, c_out):
        return 0


def test_routing_predicates(monkeypatch):
    """bn_act_conv: training → the fused BNActConv, eval + gradients → the differentiable row path (unchanged), eval
    without gradients → the split fusion; ResBlock.infer_ok follows the same predicate, and a deferred MinkowskiBatchNorm
    reaches its convolution through this route."""
    from pasco_b200 import ops
    monkeypatch.setattr(ops, "load", lambda: _NoSplitLib)
    bn = torch.nn.BatchNorm1d(64)
    x = types.SimpleNamespace(is_cuda=True)
    w = torch.empty(27, 64, 64)
    kmap = types.SimpleNamespace(K=27, nbr=object(), n_out=100_000, n_in=100_000)
    net = parity.pasconet()

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
        z = parity.fixture(f"net_cfg1_infer_{tag}.npz")
        mine = {k: list(v.shape) for k, v in parity.pasconet(M).reference_state_dict().items() if k.endswith(STAT_SUFFIXES)}
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
    assert int(parity.fixture("net_cfg1_infer_big.npz")["sem1_n"][0]) > 1_000_000


# ------------------------------------------------------------------------------------------------
# GPU: the inference epilogue against the composition of existing ops
# ------------------------------------------------------------------------------------------------
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
                with parity.launches() as launches:
                    out, nxt = ops.conv_infer(planes, W, bias_t, kmap, packs, residual=res if use_res else None,
                                              act_out=act_out, want_out=want_out, next_coefs=(sc1, sh1) if coefs else None,
                                              next_act=act_next, want_next=use_next)
                assert [x[:2] for x in launches] == [("fwd", "planes_infer")]
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
        ops.set_precision("fp32")


# ------------------------------------------------------------------------------------------------
# GPU: networks in eval mode against the eval-mode golden vectors
# ------------------------------------------------------------------------------------------------
def _stats(net):
    return {k: v.clone() for k, v in net.state_dict().items() if k.endswith(STAT_SUFFIXES + (".num_batches_tracked",))}


def _run(net, sc, fused=True):
    from pasco_b200 import ops
    ops.inference_fusion(fused)
    c0 = ops.CALLS
    try:
        with torch.no_grad(), parity.launches() as launches:
            out = parity.forward(net, sc, test=True)
        return out, ops.CALLS - c0, launches
    finally:
        ops.inference_fusion(True)


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
    ops.set_precision("fp32")
    meta = MANIFEST["cases"][f"m{M}"]
    net, gold = parity.load_eval(parity.pasconet(M), f"m{M}")
    out, calls, calls_ref = _check_fused_vs_unfused(net, parity.scene(meta, M), M)
    rep = parity.check_outputs(out, gold, meta)
    print(f"eval M={M}: C-ABI calls fused {calls} / unfused {calls_ref};", rep)


@pytest.mark.gpu
def test_pasconet_eval_benchmark_scale_matches_reference_eval_golden():
    from pasco_b200 import ops
    ops.set_precision("fp32")
    meta = MANIFEST["cases"]["big"]
    net, gold = parity.load_eval(parity.pasconet(1), "big")
    out, calls, calls_ref = _check_fused_vs_unfused(net, parity.scene(meta), 1)
    # 1.74 M decoder voxels: argmax near-ties keep ~20 scale-1 and ~3 scale-2 voxels other than the CPU run (the parent
    # engine does the same; this forward is bit-identical to it), and a flipped voxel changes the features of its
    # neighbourhood through the residual blocks, the voxel head and the attention masks.  Measured on an H100: voxel-logit
    # row error 1.4e-4 at the 95th percentile, 8e-3 at the 99th; every other output 1.2e-4 at the 99th.  Bound: the 95th
    # percentile at 1e-3 and the median at 5e-4 (test_golden_r2's near-tie rule with the cap-branch quantile's margin).
    rep = parity.check_outputs(out, gold, meta, q=0.95)
    print(f"eval benchmark scale: C-ABI calls fused {calls} / unfused {calls_ref};", rep)


def _reference_net():
    if not os.path.isdir(os.path.join(parity.REF, "pasco")):
        pytest.skip("oracle/_ref not staged")
    return parity.reference_net()


@pytest.mark.gpu
def test_unmodified_reference_eval_on_the_engine_matches_golden():
    from pasco_b200 import ops
    ops.set_precision("fp32")
    ME, net = _reference_net()
    net, gold = parity.load_eval(net, "m1", ref_names=False)
    meta = MANIFEST["cases"]["m1"]
    before = _stats(net)
    with torch.no_grad(), parity.launches() as launches:
        out = parity.forward_reference(ME, net, parity.scene(meta), torch.device("cuda"), test=True)
    assert all(torch.equal(v, _stats(net)[k]) for k, v in before.items())
    assert launches and not [x for x in launches if x[1] == "simt"]
    rep = parity.check_outputs(out, gold, meta)
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
    ops.set_precision("fp32")
    ME, net = _reference_net()
    net, _ = parity.load_eval(net, "m1", ref_names=False)
    dev = torch.device("cuda")
    sc = parity.scene(MANIFEST["cases"]["m1"])
    batch = _RecordingBatch(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                            max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                            global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                            geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"])
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
