"""The decoder hook (pasco_b200/hooks.py install(decoder=True)): the unmodified reference's DecoderBlock.forward and
DecoderGenerativeSepConvV2's predict_completion_sem_logit, predict_panop and forward on csrc/decoder.cu and
net3d.resize_rows, against the saved originals on the same inputs.

  * CPU: the new C-ABI symbols are declared and typed, no local memory in the new kernels, install / uninstall restore
    all four names;
  * GPU: pasco_completion_rows against torch (M = 1..4, K = 19 / 20, tied maxima, NaN rows); the cap against
    torch.multinomial (the exponential-race identity, the keep mask at N = 1 M and k = 400 000, the CUDA generator state
    afterwards); the M >= 3 vote cap; predict_panop bit for bit (the all-empty keep[:1000] case, unequal subnets, the
    padded batch and keep_pad); DecoderBlock.forward forward and backward in train and eval mode; every fallback
    (spied); repeats and synchronisation counts; KITTI-360 (K = 19); the unmodified Net's training and test steps with
    the other five hook groups on, decoder off and on.
GPU tests skip when oracle/_ref is not staged.
"""
import collections
import copy
import os
import re
import subprocess
import sys
import types
import warnings

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_golden_eval as GE  # noqa: E402
import parity  # noqa: E402

STAGED = os.path.isdir(os.path.join(parity.REF, "pasco"))
needs_ref = pytest.mark.skipif(not STAGED, reason="oracle/_ref not staged")
K = 20
NEW_SYMBOLS = ("pasco_completion_rows", "pasco_topk_mask", "pasco_panop_crop", "pasco_mimo_batch")
KERNELS = ("k_completion_rows", "k_labelled", "k_sel_init", "k_sel_hist", "k_sel_pick", "k_tie_counts", "k_tie_scan",
           "k_topk_write", "k_crop", "k_crop_empty", "k_mimo_batch")
PATCHED = (("DecoderBlock", "forward"), ("DecoderGenerativeSepConvV2", "predict_completion_sem_logit"),
           ("DecoderGenerativeSepConvV2", "predict_panop"), ("DecoderGenerativeSepConvV2", "forward"))


# ------------------------------------------------------------------------------------------------
# CPU
# ------------------------------------------------------------------------------------------------
def test_new_symbols_declared_and_typed():
    from pasco_b200 import _lib
    src = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pasco_sm100.h")).read(), flags=re.S)
    for name in NEW_SYMBOLS:
        m = re.search(r"\b" + name + r"\s*\(([^;)]*)\)\s*;", src)
        assert m, f"{name} not declared"
        n_args = len([a for a in m.group(1).split(",") if a.strip()])
        assert name in _lib.PROTOTYPES and len(_lib.PROTOTYPES[name][1]) == n_args, name


def test_new_kernels_use_no_local_memory():
    from pasco_b200 import _lib, build
    build.build()
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout
    found = collections.Counter()
    for f in re.split(r"\n\s*Function : ", sass):
        head = f.split("\n")[0]
        if "decoder_cu" not in head:
            continue
        for n in KERNELS:
            if re.search(r"\d" + n + r"(E|I)", head):
                found[n] += 1
                assert not re.search(r"\b(LDL|STL)\b", f), f"{head}: local-memory traffic"
    assert set(found) == set(KERNELS), set(KERNELS) - set(found)


def _decoder_module():
    parity.reference_net()
    import importlib
    return importlib.import_module("pasco.models.decoder_v3")


@needs_ref
def test_install_uninstall_restores_the_four_names():
    from pasco_b200 import hooks
    d = _decoder_module()
    names = lambda: tuple(getattr(getattr(d, c), n) for c, n in PATCHED)  # noqa: E731
    before = names()
    assert hooks.install(attention=False, trunk=True)
    assert names() == before                                            # not requested: untouched
    for _ in range(2):
        assert hooks.install(attention=False, decoder=True)
    assert names() == (hooks._decoder_block_forward, hooks._predict_completion_sem_logit, hooks._predict_panop,
                       hooks._decoder_forward)
    for (c, n), fn in zip(PATCHED, before):
        assert getattr(getattr(d, c), "_pasco_b200_orig_" + n) is fn
    for _ in range(2):
        hooks.uninstall()
    assert names() == before


# ------------------------------------------------------------------------------------------------
# GPU: pasco_completion_rows
# ------------------------------------------------------------------------------------------------
def _logits(n, k, g, ties=True, nans=True):
    L = torch.randn(n, k, generator=g)
    if ties:
        L[::5, 3] = L[::5, 7] = 4.0                  # tied maxima: the first index wins
        L[1::7, 0] = L[1::7, 2] = 5.0
        L[2::11] = 1.0                               # a whole row tied
    if nans:
        L[3::13, 5] = float("nan")                   # a NaN wins at its first index
        L[4::17, 0] = float("nan")
    return L.cuda()


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2, 3, 4])
@pytest.mark.parametrize("Kc", [19, 20])
def test_completion_rows_match_torch(M, Kc):
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(M * 100 + Kc)
    n = 50_000
    probs = [torch.softmax(_logits(n, Kc, g), -1) for _ in range(M)]
    probs[0][6::19] = 1.0 / Kc                                         # equal probabilities in a row
    w = torch.rand(Kc, generator=g).cuda() + 0.5
    labels = [torch.randint(0, 256, (32, 32, 4), generator=g).to(torch.uint8).cuda() for _ in range(M)]
    cls, keep, weight, votes, counts = ops.completion_rows(probs, w, labels)
    want_keep = []
    for m, p in enumerate(probs):
        pm, cm = p.max(-1)
        assert torch.equal(cls[m].long(), cm)
        assert torch.equal(keep[m], cm != 0)
        assert torch.equal(weight[m].view(torch.int32), (pm * w[cm]).view(torch.int32))
        want_keep.append(cm != 0)
    assert (torch.stack([p.isnan().any(-1) for p in probs])).any()
    want_votes = torch.stack(want_keep).sum(0)
    assert torch.equal(votes.long(), want_votes)
    want_counts = ([int(k.sum()) for k in want_keep] + [int(((t != 0) & (t != 255)).sum()) for t in labels]
                   + [int((~((weight[m] >= 0) & weight[m].isfinite())).sum()) for m in range(M)]
                   + [int((want_votes > 0).sum())])
    assert counts.tolist() == want_counts
    assert sum(counts.tolist()[2 * M:3 * M]) > 0                      # the NaN rows are counted as bad weights


# ------------------------------------------------------------------------------------------------
# GPU: the cap
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("k", [1000, 40_000])
def test_multinomial_is_topk_over_exponential_on_cuda(k):
    w = torch.rand(100_000, generator=torch.Generator().manual_seed(k)).cuda()
    torch.cuda.manual_seed(7)
    want = torch.multinomial(w, k, replacement=False)
    after_want = torch.cuda.get_rng_state()
    torch.cuda.manual_seed(7)
    q = torch.empty_like(w).exponential_(1)
    got = torch.topk(w / q, k)[1]
    assert torch.equal(got, want)
    assert torch.equal(torch.cuda.get_rng_state(), after_want)


def _decoder(d, M, training):
    D = d.DecoderGenerativeSepConvV2
    dec = D.__new__(D)
    torch.nn.Module.__init__(dec)
    dec.n_infers = M
    dec.occ_thres = {1: {4: 25000, 2: 120000, 1: 400000}, 2: {4: 25000, 2: 120000, 1: 400000},
                     3: {4: 24000, 2: 100000, 1: 350000}, 4: {4: 22000, 2: 80000, 1: 320000}}[M]
    dec.agg_occ_thres = {4: 30000, 2: 100000, 1: 400000}
    dec.pruning = d.ME.MinkowskiPruning()
    dec.train(training)
    return dec


def _completion_inputs(M, n, scale, seed, empty_bias=0.0):
    g = torch.Generator().manual_seed(seed)
    sem = []
    for _ in range(M):
        L = torch.randn(n, K, generator=g)
        L[:, 0] += empty_bias
        L[::3, 4] = L[::3, 9] = 6.0                   # many bit-identical weights
        sem.append(types.SimpleNamespace(F=L.cuda()))
    x = types.SimpleNamespace(C=torch.zeros(n, 4, dtype=torch.int32, device="cuda"))
    labels = {f"1_{scale}": torch.randint(0, 21, (M, 64, 64, 8), generator=g).to(torch.uint8).cuda()}
    labels[f"1_{scale}"][:, :4] = 255
    freqs = {f"1_{scale}": np.random.default_rng(seed).uniform(1e3, 1e6, K)}
    return x, sem, labels, freqs


def _both_keeps(d, dec, x, scale, sem, labels, freqs, test, capsys, seed=11):
    out = []
    for fn in (d.DecoderGenerativeSepConvV2._pasco_b200_orig_predict_completion_sem_logit,
               d.DecoderGenerativeSepConvV2.predict_completion_sem_logit):
        torch.cuda.manual_seed(seed)
        capsys.readouterr()
        keep = fn(dec, x, scale, sem, None, [None] * len(sem), [None] * len(sem), freqs, sem_labels=labels, test=test)
        out.append((keep, torch.cuda.get_rng_state(), capsys.readouterr().out))
    return out


@pytest.fixture
def dec_hooks():
    from pasco_b200 import hooks
    d = _decoder_module()
    import MinkowskiEngine as ME
    d.ME = ME
    hooks.uninstall()
    assert hooks.install(attention=False, decoder=True)
    try:
        yield d
    finally:
        hooks.uninstall()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_cap_matches_multinomial_at_full_size(dec_hooks, M, capsys):
    d = dec_hooks
    n = 1_050_000
    x, sem, labels, freqs = _completion_inputs(M, n, 1, seed=M)
    (k0, r0, p0), (k1, r1, p1) = _both_keeps(d, _decoder(d, M, True), x, 1, sem, labels, freqs, False, capsys)
    assert int(k1.sum()) >= 400_000 and p0.count("Scale 1, infer") == M
    assert torch.equal(r0, r1), "the CUDA generator moved differently"
    assert p0 == p1
    diff = int((k0 != k1).sum())
    print(f"M = {M}: {diff} rows differ of {n}")
    assert torch.equal(k0, k1)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("scale,n,training", [(4, 100_000, False), (1, 600_000, True), (2, 1000, True)])
def test_vote_cap_matches_the_original(dec_hooks, scale, n, training, capsys):
    """M = 3: the union above agg_occ_thres (torch.topk over the votes), a per-subnet cap above 500 000 rows first, and
    a union of at most 2 rows (keep all but the cap's top-k over votes that are all 0)."""
    d = dec_hooks
    x, sem, labels, freqs = _completion_inputs(3, n, scale, seed=scale, empty_bias=30.0 if n == 1000 else 0.0)
    if n == 1000:
        sem[1].F[5, 7] = 100.0
        for fn in (d.DecoderGenerativeSepConvV2._pasco_b200_orig_predict_completion_sem_logit,
                   d.DecoderGenerativeSepConvV2.predict_completion_sem_logit):
            with pytest.raises(RuntimeError):           # k = 100 000 > n rows: the original's error, unchanged
                fn(_decoder(d, 3, training), x, scale, sem, None, [None] * 3, [None] * 3, freqs, sem_labels=labels)
        return
    (k0, r0, p0), (k1, r1, p1) = _both_keeps(d, _decoder(d, 3, training), x, scale, sem, labels, freqs, False, capsys)
    assert "Overall keep" in p0 and p0 == p1
    assert torch.equal(k0, k1) and torch.equal(r0, r1)
    (t0, _, q0), (t1, _, q1) = _both_keeps(d, _decoder(d, 3, training), x, scale, sem, labels, freqs, True, capsys)
    assert torch.equal(t0, t1) and q0 == q1 == ""


# ------------------------------------------------------------------------------------------------
# GPU: predict_panop
# ------------------------------------------------------------------------------------------------
def _voxel_feats(ME, scales, M, ch):
    torch.manual_seed(3)
    return torch.nn.ModuleDict({f"scale{s}_infer{m}": torch.nn.Sequential(
        ME.MinkowskiConvolution(ch[s], ch[s], kernel_size=3, bias=False, dimension=3), ME.MinkowskiBatchNorm(ch[s]),
        ME.MinkowskiReLU(), ME.MinkowskiConvolution(ch[s], ch[s], kernel_size=3, bias=True, dimension=3))
        for s in scales for m in range(M)}).cuda()


def _panop_inputs(ME, M, seed, Kc=K, n1=6000, empty=True):
    g = torch.Generator().manual_seed(seed)
    ch = {4: 128, 2: 64, 1: 64}
    xs, sem = {}, {}
    for s, n in ((4, n1 // 8), (2, n1 // 3), (1, n1)):
        cells = torch.unique(torch.randint(-10, 40, (n, 3), generator=g), dim=0) * s
        C = torch.cat([torch.zeros(cells.shape[0], 1, dtype=torch.long), cells], 1).int().cuda()
        x = ME.SparseTensor(torch.randn(C.shape[0], ch[s], generator=g).cuda(), C, tensor_stride=s)
        xs[s] = x
        sem[s] = []
        for m in range(M):
            L = torch.randn(C.shape[0], Kc, generator=g)
            L[:, 0] += 1.5 * m
            if empty and m == M - 1 and s == 4:
                L[:, 0] = 50.0                        # no row with a non-empty argmax: keep[:1000], then the box
            sem[s].append(ME.SparseTensor(L.cuda(), coordinate_map_key=x.coordinate_map_key,
                                          coordinate_manager=x.coordinate_manager))
    min_Cs = [torch.tensor([-8 + 4 * m, -10, 0], device="cuda") for m in range(M)]
    max_Cs = [torch.tensor([30, 25 - 3 * m, 150], device="cuda") for m in range(M)]
    labels = {f"1_{s}": torch.zeros(M, 4, 4, 4, dtype=torch.uint8, device="cuda") for s in (1, 2, 4)}
    return xs, sem, min_Cs, max_Cs, labels, ch


class _Recorder(torch.nn.Module):
    """Stands in for transformer_predictor: keeps the inputs it is given."""

    def __init__(self):
        super().__init__()
        self.got = None

    def forward(self, xs, sem, min_Cs, max_Cs, keep_pad):
        self.got = ({s: (f.detach().clone(), c.clone()) for s, (f, c) in xs.items()},
                    (sem[0].detach().clone(), sem[1].clone()), keep_pad.clone())
        return "preds"


def _panop_both(d, M, inputs, capsys, voxel_feats=None):
    xs, sem, min_Cs, max_Cs, labels, ch = inputs
    ME = d.ME
    base = _decoder(d, M, True)
    base.voxel_feats = voxel_feats if voxel_feats is not None else _voxel_feats(ME, (4, 2, 1), M, ch)
    out = []
    for fn in (d.DecoderGenerativeSepConvV2._pasco_b200_orig_predict_panop, d.DecoderGenerativeSepConvV2.predict_panop):
        dec = copy.deepcopy(base)
        rec = _Recorder()
        dec.transformer_predictor = rec
        capsys.readouterr()
        preds, pruned = fn(dec, xs, sem, None, min_Cs, max_Cs, labels)
        out.append((preds, [(p.F.detach(), p.C) for p in pruned], rec.got, capsys.readouterr().out))
    return out


def _bits_equal(a, b):
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.contiguous().view(torch.uint8),
                                                                      b.contiguous().view(torch.uint8))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2, 3])
def test_predict_panop_bit_identical(dec_hooks, M, capsys):
    d = dec_hooks
    (p0, s0, r0, o0), (p1, s1, r1, o1) = _panop_both(d, M, _panop_inputs(d.ME, M, seed=M), capsys)
    assert p0 == p1 == "preds"
    assert o0 == o1 and o0.count("line 367") == 1
    assert len(s0) == len(s1) == M
    for (f0, c0), (f1, c1) in zip(s0, s1):
        assert _bits_equal(f0, f1) and torch.equal(c0, c1)
    xs0, (bf0, bc0), kp0 = r0
    xs1, (bf1, bc1), kp1 = r1
    assert list(xs0) == list(xs1) == [4, 2, 1]
    for s in xs0:
        assert _bits_equal(xs0[s][0], xs1[s][0]) and _bits_equal(xs0[s][1], xs1[s][1]), f"scale {s}"
    assert _bits_equal(bf0, bf1) and _bits_equal(bc0, bc1) and _bits_equal(kp0, kp1)
    if M > 1:
        assert len({f.shape[0] for f, _ in s0}) > 1                    # subnets of unequal length: padded rows
        assert not kp0.all()


@pytest.mark.gpu
@needs_ref
def test_mimo_batch_matches_batch_sparse_tensor(dec_hooks):
    """Features, coordinates and keep_pad against utils.py:659-670 and decoder_v3.py:443-446, with keep_pad's own rule
    (any feature or coordinate != 0), not "row < length": a real row whose logits and coordinates are all zero is dropped,
    −0.0 counts as zero and a NaN as non-zero."""
    from pasco.models.utils import batch_sparse_tensor
    from pasco_b200 import ops
    g = torch.Generator().manual_seed(8)
    rows = []
    for n in (700, 1200, 0, 950):
        F_ = torch.randn(n, K, generator=g)
        C_ = torch.randint(-20, 20, (n, 4), generator=g).int()
        if n:
            F_[3], C_[3] = 0.0, 0                      # a real all-zero row
            F_[5], C_[5] = -0.0, 0
            F_[7, 2], C_[7] = float("nan"), 0
        rows.append(types.SimpleNamespace(F=F_.cuda().requires_grad_(True), C=C_.cuda(), shape=F_.shape))
    want_F, want_C = batch_sparse_tensor(rows)
    want_keep = ((want_F != 0).sum(-1) + (want_C != 0).sum(-1)) != 0
    got_F, got_C, got_keep = ops.mimo_batch([r.F for r in rows], [r.C for r in rows], keep_pad=True)
    assert _bits_equal(got_F.detach(), want_F.detach()) and _bits_equal(got_C, want_C)
    assert torch.equal(got_keep, want_keep) and not got_keep[0, 3] and not got_keep[0, 5] and got_keep[0, 7]
    w = torch.randn(want_F.shape, generator=g).cuda()
    ga = torch.autograd.grad((want_F * w).nansum(), [r.F for r in rows if r.F.shape[0]])
    gb = torch.autograd.grad((got_F * w).nansum(), [r.F for r in rows if r.F.shape[0]])
    assert all(_bits_equal(a_, b_) for a_, b_ in zip(ga, gb))


# ------------------------------------------------------------------------------------------------
# GPU: DecoderBlock.forward
# ------------------------------------------------------------------------------------------------
def _block(d, cin, cout, train, heads=2, Kc=K, dropout=0.0):
    from pasco.models.dropout import MinkowskiSpatialDropout
    torch.manual_seed(5)
    blk = d.DecoderBlock(cin, cout, dropout_layer=MinkowskiSpatialDropout, scene_size=(256, 256, 32),
                         drop_path_rates=[0.0] * 7, n_heads=heads, compl_head_dim=Kc, heavy_decoder=dropout > 0,
                         dropout=dropout).cuda()
    for m in blk.modules():
        if isinstance(m, torch.nn.BatchNorm1d):
            m.weight.data.uniform_(0.5, 1.5)
            m.bias.data.uniform_(-0.2, 0.2)
            m.running_mean.uniform_(-0.1, 0.1)
            m.running_var.uniform_(0.5, 2.0)
    return blk.train(train)


def _block_inputs(ME, cin, cout, seed, n=4000):
    g = torch.Generator().manual_seed(seed)
    cells = torch.unique(torch.randint(-6, 30, (n, 3), generator=g), dim=0) * 2
    C = torch.cat([torch.zeros(cells.shape[0], 1, dtype=torch.long), cells], 1).int().cuda()
    cm = ME.CoordinateManager()
    Fx = torch.randn(C.shape[0], cin, generator=g).cuda()
    sc = torch.unique(torch.randint(-12, 60, (3 * n, 3), generator=g), dim=0)
    Cs = torch.cat([torch.zeros(sc.shape[0], 1, dtype=torch.long), sc], 1).int().cuda()
    Fs = torch.randn(Cs.shape[0], cout, generator=g).cuda()
    gmin, gmax = torch.tensor([-4, -8, 0], device="cuda"), torch.tensor([50, 47, 55], device="cuda")
    return Fx, C, Fs, Cs, cm, gmin, gmax


def _block_run(ME, blk, fn, inputs):
    Fx, C, Fs, Cs, _, gmin, gmax = inputs
    cm = ME.CoordinateManager()
    x = Fx.clone().requires_grad_(True)
    s = Fs.clone().requires_grad_(True)
    xt = ME.SparseTensor(x, C, tensor_stride=2, coordinate_manager=cm)
    st = ME.SparseTensor(s, Cs, tensor_stride=1, coordinate_manager=cm)
    blk.zero_grad(set_to_none=True)
    h, logits = fn(blk, xt, st, gmin, gmax)
    g = torch.Generator().manual_seed(1)
    loss = (h.F * torch.randn(h.F.shape, generator=g).cuda()).sum()
    for lg in logits:
        loss = loss + (lg.F * torch.randn(lg.F.shape, generator=g).cuda()).sum()
    loss.backward()
    grads = {n: p.grad.detach().clone() for n, p in blk.named_parameters() if p.grad is not None}
    grads["x"], grads["shortcut"] = x.grad, s.grad
    return h.F.detach(), h.C, [lg.F.detach() for lg in logits], grads


def _maxabs(a, b):
    return float((a.double() - b.double()).abs().max() / b.double().abs().max().clamp(min=1e-30))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("train", [True, False])
def test_decoder_block_matches_the_original(dec_hooks, train):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    d = dec_hooks
    inputs = _block_inputs(d.ME, 128, 64, seed=2)
    base = _block(d, 128, 64, train)
    want = _block_run(d.ME, copy.deepcopy(base), d.DecoderBlock._pasco_b200_orig_forward, inputs)
    got = _block_run(d.ME, copy.deepcopy(base), d.DecoderBlock.forward, inputs)
    assert torch.equal(got[1], want[1])                                # same rows, same order
    assert _maxabs(got[0], want[0]) < 1e-3
    for a, b in zip(got[2], want[2]):
        assert _maxabs(a, b) < 1e-3
    assert set(got[3]) == set(want[3])
    rel = {n: float((got[3][n] - want[3][n]).double().norm() / want[3][n].double().norm().clamp(min=1e-30))
           for n in want[3]}
    print("worst gradients (relative L2):", sorted(rel.items(), key=lambda kv: -kv[1])[:4])
    assert max(rel.values()) < 1e-2, rel


# ------------------------------------------------------------------------------------------------
# GPU: fallbacks
# ------------------------------------------------------------------------------------------------
def _spy(cls, attr, calls):
    orig = getattr(cls, attr)
    setattr(cls, attr, lambda *a, **k: calls.append(attr) or "orig")
    return orig


def _spied(cls, attr, run):
    calls = []
    orig = _spy(cls, attr, calls)
    try:
        out = run()
    finally:
        setattr(cls, attr, orig)
    return calls == [attr] and out == "orig"


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "nine_subnets", "k65", "fp64", "no_labels"])
def test_completion_fallbacks(dec_hooks, case):
    d = dec_hooks
    M = 9 if case == "nine_subnets" else 2
    x, sem, labels, freqs = _completion_inputs(M, 2000, 4, seed=0)
    if case == "cpu":
        sem = [types.SimpleNamespace(F=s.F.cpu()) for s in sem]
    if case == "k65":
        sem = [types.SimpleNamespace(F=torch.randn(2000, 65, device="cuda")) for _ in sem]
    if case == "fp64":
        sem = [types.SimpleNamespace(F=s.F.double()) for s in sem]
    dec = _decoder(d, min(M, 4), True)
    dec.n_infers = M
    D = d.DecoderGenerativeSepConvV2
    assert _spied(D, "_pasco_b200_orig_predict_completion_sem_logit",
                  lambda: D.predict_completion_sem_logit(dec, x, 4, sem, None, None, None, freqs,
                                                         sem_labels=None if case == "no_labels" else labels))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "nine_subnets", "k65", "fp64", "box_float", "separate_maps"])
def test_panop_fallbacks(dec_hooks, case):
    d = dec_hooks
    ME = d.ME
    M = 9 if case == "nine_subnets" else 2
    xs, sem, min_Cs, max_Cs, labels, ch = _panop_inputs(ME, M, seed=4, n1=800)
    if case == "cpu":
        xs = {s: types.SimpleNamespace(F=x.F.cpu(), C=x.C.cpu(), coordinate_map_key=x.coordinate_map_key)
              for s, x in xs.items()}
    if case in ("k65", "fp64"):
        for s in sem:
            t = sem[s][0]
            F_ = torch.randn(t.F.shape[0], 65, device="cuda") if case == "k65" else t.F.double()
            sem[s][0] = types.SimpleNamespace(F=F_, C=t.C, coordinate_map_key=t.coordinate_map_key)
    if case == "box_float":
        min_Cs[0] = min_Cs[0].float()
    if case == "separate_maps":
        sem[2][1] = ME.SparseTensor(sem[2][1].F, sem[2][1].C.clone(), tensor_stride=2)
    dec = _decoder(d, min(M, 4), True)
    dec.n_infers = M
    D = d.DecoderGenerativeSepConvV2
    assert _spied(D, "_pasco_b200_orig_predict_panop",
                  lambda: D.predict_panop(dec, xs, sem, None, min_Cs, max_Cs, labels))


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("case", ["cpu", "not_the_pair", "c_not_64_train", "dropout_train", "decoder_forward_cpu"])
def test_block_and_forward_fallbacks(dec_hooks, case):
    d = dec_hooks
    ME = d.ME
    if case == "decoder_forward_cpu":
        D = d.DecoderGenerativeSepConvV2
        x = types.SimpleNamespace(F=torch.zeros(3, 4))
        assert _spied(D, "_pasco_b200_orig_forward",
                      lambda: D.forward(_decoder(d, 1, True), x, [], None, None, None, None, None, None))
        return
    cout = 48 if case == "c_not_64_train" else 64
    blk = _block(d, 128, cout, True, dropout=0.3 if case == "dropout_train" else 0.0)
    if case == "not_the_pair":
        blk.resize = torch.nn.Sequential(blk.resize[0], ME.MinkowskiConvolution(cout + 3, cout, kernel_size=3,
                                                                                 bias=True, dimension=3).cuda())
    Fx, C, Fs, Cs, cm, gmin, gmax = _block_inputs(ME, 128, cout, seed=1, n=500)
    if case == "cpu":
        xt = types.SimpleNamespace(F=Fx.cpu())
        st = None
    else:
        xt = ME.SparseTensor(Fx, C, tensor_stride=2, coordinate_manager=cm)
        st = ME.SparseTensor(Fs, Cs, coordinate_manager=cm)
    B = d.DecoderBlock
    assert _spied(B, "_pasco_b200_orig_forward", lambda: B.forward(blk, xt, st, gmin, gmax))
    if case in ("c_not_64_train", "dropout_train"):        # eval mode: the hook runs
        blk.eval()
        calls = []
        orig = _spy(B, "_pasco_b200_orig_forward", calls)
        try:
            B.forward(blk, xt, st, gmin, gmax)
        finally:
            B._pasco_b200_orig_forward = orig
        assert calls == []


# ------------------------------------------------------------------------------------------------
# GPU: repeats and host synchronisations
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
def test_repeats_bit_identical_and_syncs_constant(dec_hooks, capsys):
    from pasco_b200 import hooks
    d = dec_hooks
    D = d.DecoderGenerativeSepConvV2
    counts = collections.defaultdict(set)
    for M, n, seed in ((2, 200_000, 1), (3, 600_000, 2)):
        x, sem, labels, freqs = _completion_inputs(M, n, 1, seed=seed)
        dec = _decoder(d, M, True)
        inputs = _panop_inputs(d.ME, M, seed=seed, n1=3000 * M)
        ident = torch.nn.ModuleDict({f"scale{s}_infer{m}": torch.nn.Identity() for s in (4, 2, 1) for m in range(M)})
        outs = []
        for _ in range(2):
            torch.cuda.manual_seed(3)
            keep, s1 = _syncs(lambda: D.predict_completion_sem_logit(dec, x, 1, sem, None, None, None, freqs,
                                                                     sem_labels=labels))
            dec.voxel_feats, dec.transformer_predictor = ident, _Recorder()
            (_, pruned), s2 = _syncs(lambda: D.predict_panop(dec, *inputs[:1], inputs[1], None, *inputs[2:5]))
            counts["predict_completion_sem_logit", M].add(tuple(s1))
            counts["predict_panop", M].add(tuple(s2))
            outs.append([keep] + [p.F for p in pruned] + [t for s, (f, c) in dec.transformer_predictor.got[0].items()
                                                          for t in (f, c)] + [dec.transformer_predictor.got[2]])
        for a_, b_ in zip(*outs):
            assert _bits_equal(a_, b_)
    capsys.readouterr()
    print("host synchronisations per hooked call:", dict(counts))
    for k, v in counts.items():
        assert len(v) == 1 and len(next(iter(v))) <= hooks.DECODER_SYNCS, (k, v)
    assert counts["predict_panop", 2] == counts["predict_panop", 3]


# ------------------------------------------------------------------------------------------------
# GPU: KITTI-360 (K = 19) goes through the hooked path
# ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@needs_ref
def test_kitti360_decoder_takes_the_hooked_path(dec_hooks, capsys):
    from pasco.models.net_panoptic_sparse_kitti360 import Net_kitti360
    d = dec_hooks
    torch.manual_seed(0)
    net = Net_kitti360(n_classes=19, class_names=[str(i) for i in range(19)], class_weights=torch.ones(19),
                       encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3, dense3d_dropout=0.0, n_infers=2,
                       class_frequencies={f"1_{s}": np.ones(19) for s in (1, 2, 4)}, in_channels=8, f=64).cuda().train()
    dg = net.unet3d.decoder_generative
    assert type(dg) is d.DecoderGenerativeSepConvV2 and all(type(b) is d.DecoderBlock for b in dg.dec_blocks)
    calls = []
    saved = [(c, n, _spy(getattr(d, c), "_pasco_b200_orig_" + n, calls)) for c, n in PATCHED]
    try:
        x, sem, labels, freqs = _completion_inputs(2, 30_000, 4, seed=19)
        freqs = {k: v[:19] for k, v in freqs.items()}
        for s in sem:
            s.F = s.F[:, :19].contiguous()
        keep = dg.predict_completion_sem_logit(x, 4, sem, None, None, None, freqs, sem_labels=labels)
        xs, semp, lo, hi, lab, ch = _panop_inputs(d.ME, 2, seed=19, Kc=19)
        rec = _Recorder()
        dg.transformer_predictor = rec
        dg.voxel_feats = _voxel_feats(d.ME, (4, 2, 1), 2, ch)
        dg.predict_panop(xs, semp, None, lo, hi, lab)
        blk = _block(d, 128, 64, True, Kc=19)
        Fx, C, Fs, Cs, cm, gmin, gmax = _block_inputs(d.ME, 128, 64, seed=3, n=800)
        h, logits = blk(d.ME.SparseTensor(Fx, C, tensor_stride=2, coordinate_manager=cm),
                        d.ME.SparseTensor(Fs, Cs, coordinate_manager=cm), gmin, gmax)
    finally:
        for c, n, orig in saved:
            setattr(getattr(d, c), "_pasco_b200_orig_" + n, orig)
    assert calls == []
    assert keep.dtype == torch.bool and rec.got is not None and logits[0].F.shape[1] == 19


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified Net end to end, the other five hook groups on
# ------------------------------------------------------------------------------------------------
class _Coords:
    """The coordinate sets the transformer receives at every decoder scale, per call."""

    def __init__(self):
        from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
        self.cls, self.got = TransformerPredictorV2, []

    def __enter__(self):
        inner = self.cls.forward

        def rec(this, xs, *a, **k):
            self.got.append({s: np.unique(xs[s][1].reshape(-1, 4).cpu().numpy(), axis=0) for s in xs})
            return inner(this, xs, *a, **k)
        self.inner = inner
        self.cls.forward = rec
        return self

    def __exit__(self, *exc):
        self.cls.forward = self.inner


def _set(hooks, decoder):
    hooks.uninstall()
    assert hooks.install(attention=True, postprocess=True, evaluate=True, criterion=True, trunk=True, decoder=decoder)


def _same_coords(a, b):
    assert len(a) == len(b)
    for x, y in zip(a, b):
        assert set(x) == set(y)
        for s in x:
            assert np.array_equal(x[s], y[s]), f"scale {s}"


def _val(v):
    return float(v.detach()) if torch.is_tensor(v) else float(v)


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_net_training_step_decoder_off_and_on(M, capsys):
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

    def step(decoder):
        _set(hooks, decoder)
        net.load_state_dict(state)
        logged = {}
        net.log = lambda k, v, **kw: logged.__setitem__(k, _val(v))
        net.zero_grad(set_to_none=True)
        torch.manual_seed(0)
        capsys.readouterr()
        with _Coords() as rec:
            out = net.step(batch, "train")
        out["loss"].backward()
        grads = {n: p.grad.detach().clone() for n, p in net.named_parameters() if p.grad is not None}
        return _val(out["loss"]), logged, rec.got, grads, capsys.readouterr().out

    try:
        want = step(False)
        got = step(True)
    finally:
        hooks.uninstall()
    _same_coords(got[2], want[2])
    assert got[4] == want[4]
    assert set(got[1]) == set(want[1])
    for k, v in want[1].items():
        assert abs(got[1][k] - v) <= 1e-3 * max(1.0, abs(v)), (k, got[1][k], v)
    assert set(got[3]) == set(want[3])
    num = sum(float((got[3][n] - want[3][n]).double().norm() ** 2) for n in want[3]) ** 0.5
    den = sum(float(want[3][n].double().norm() ** 2) for n in want[3]) ** 0.5
    print(f"M = {M}: loss {got[0]:.6f} (decoder on) vs {want[0]:.6f} (off); gradients relative L2 {num / den:.2e}")
    assert num / den < 1e-2


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 3])
def test_net_step_inference_decoder_off_and_on(M, capsys):
    from pasco_b200 import hooks, ops
    from recipe import fill_state_dict
    ops.set_precision("fp32")
    hooks.uninstall()
    _, net = parity.reference_net(n_infers=M)
    if M == 1:
        net, _ = parity.load_eval(net, "m1", ref_names=False)
    else:
        net.load_state_dict(fill_state_dict(net.state_dict()))
        net.cuda().eval()
    net.object_mask_threshold = 0.05
    dev = torch.device("cuda")
    sc = parity.scene(parity.INFER_MANIFEST["cases"]["m1"], M)
    sem, ml = GE.gt_scene(0)
    ml = {"labels": ml["labels"].to(dev), "masks": ml["masks"].to(dev)}
    batch = dict(in_feats=sc["in_feats"], in_coords=sc["in_coords"], min_Cs=[t.to(dev) for t in sc["min_Cs"]],
                 max_Cs=[t.to(dev) for t in sc["max_Cs"]], Ts=[t.to(dev) for t in sc["Ts"]],
                 global_min_Cs=sc["global_min_Cs"].to(dev), global_max_Cs=sc["global_max_Cs"].to(dev),
                 geo_labels=sc["sem_labels"], mask_classes=sc["mask_classes"],
                 semantic_label=sem.unsqueeze(0).to(dev), semantic_label_origin=sem.unsqueeze(0).to(dev),
                 mask_label=[ml], mask_label_origin=[ml])
    from pasco.loss.panoptic_quality import PQStat
    from pasco.models.metrics import SSCMetrics, UncertaintyMetrics

    def run(decoder):
        _set(hooks, decoder)
        for i in net.pq_stat["test"]:
            net.pq_stat["test"][i] = PQStat()
            net.ssc_metrics["test"][i] = SSCMetrics(net.n_classes)
            net.uncertainty_metrics["test"][i] = UncertaintyMetrics()
            net.uncertainty_metrics_by_thresholds[0.5][i] = UncertaintyMetrics()
        torch.manual_seed(0)
        capsys.readouterr()
        with _Coords() as rec, torch.no_grad():
            net.step_inference(batch, "test", eval=True)
        ssc = {i: (m.completion_tp, m.completion_fp, m.completion_fn, m.tps.tolist())
               for i, m in net.ssc_metrics["test"].items()}
        pq = {i: {c: (s.tp, s.fp, s.fn) for c, s in p.pq_per_cat.items()} for i, p in net.pq_stat["test"].items()}
        return rec.got, ssc, pq, capsys.readouterr().out

    try:
        want = run(False)
        got = run(True)
    finally:
        hooks.uninstall()
    _same_coords(got[0], want[0])
    assert got[1] == want[1]
    assert got[2] == want[2]
    assert got[3] == want[3]
