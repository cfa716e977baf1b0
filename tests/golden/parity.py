"""The golden fixtures' two formats, written and read here only, and the setup the parity tests share.

rows     (make_golden.py, make_golden_widths.py, make_golden_queries.py): `<name>_C` the coordinates in key order (int16),
         `<name>_F` every `step`-th feature row in that order, `<name>_sum` Σ / Σ|·| over all rows.
summary  (make_golden_r2.py, make_golden_infer.py): `<name>_n` the row count, `<name>_ksum` the wrap-around key sum and xor
         (bit-exact coordinate set identity), `<name>_Fsum` Σ / Σ|·| / max|·|, `<name>_subK` / `<name>_subF` every
         `step`-th key and feature row in key order.
Both store the query logits of the final and the three auxiliary levels as `query_logits<sfx>` / `aux<i>_query_logits<sfx>`,
and name the outputs `sem<s><sfx>` / `vox<sfx>`, with sfx = "" at M = 1 and "_m<m>" at M > 1.

Only numpy and torch are imported at load time (pasco_b200, the CPU oracle and the reference inside the functions that
use them), so the CPU tests, the GPU tests and the generators all import this module.
"""
import contextlib
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
REF = os.path.join(ROOT, "oracle", "_ref")     # the unmodified reference, staged by build() when a checkout was readable

TOL_FP32 = 1e-3      # north_star tolerance for fp32 features
TOL_TIGHT = 2e-5     # what bf16x3 / fp32 SIMT actually deliver
TOL_BF16 = 2e-2      # bf16 operands (SURVEY.md §8c item 4)


def keys(C):
    """(b, x, y, z) rows → int64 keys whose order is the rows' lexicographic order."""
    c = torch.as_tensor(C).long().cpu()
    return ((c[:, 0] + 32768) << 48) | ((c[:, 1] + 32768) << 32) | ((c[:, 2] + 32768) << 16) | (c[:, 3] + 32768)


def _sfx(m, n_infers):
    return "" if n_infers == 1 else f"_m{m}"


# ------------------------------------------------------------------------------------------------
# writers
# ------------------------------------------------------------------------------------------------
def rows(arrays, name, C, F, step):
    order = torch.argsort(keys(C))
    f = F.detach().cpu()[order].numpy()
    arrays[f"{name}_C"] = C.cpu()[order].numpy().astype(np.int16)
    arrays[f"{name}_F"] = f[::step]
    arrays[f"{name}_sum"] = np.array([f.sum(dtype=np.float64), np.abs(f).sum(dtype=np.float64)])


def summary(arrays, name, C, F, step):
    k = keys(C)
    order = torch.argsort(k)
    k, F = k[order], F.detach().cpu()[order]
    kn = k.numpy()
    arrays[f"{name}_n"] = np.array([len(kn)], dtype=np.int64)
    arrays[f"{name}_ksum"] = np.array([np.add.reduce(kn.astype(np.uint64)), np.bitwise_xor.reduce(kn.astype(np.uint64))], dtype=np.uint64)
    arrays[f"{name}_Fsum"] = np.array([F.double().sum().item(), F.double().abs().sum().item(), F.abs().max().item()])
    arrays[f"{name}_subK"] = kn[::step]
    arrays[f"{name}_subF"] = F[::step].numpy()


def collect(out, n_infers, step, arrays, writer):
    """Every output of every subnet: `writer` (rows or summary) for the semantic and voxel logits, the query logits as
    they are."""
    for m in range(n_infers):
        sfx = _sfx(m, n_infers)
        for s, lg in out["sem_logits_at_scales"].items():
            writer(arrays, f"sem{s}{sfx}", lg[m].C, lg[m].F, step)
        p = out["panop_predictions"][m]
        writer(arrays, f"vox{sfx}", p["voxel_logits"].C, p["voxel_logits"].F, step)
        arrays[f"query_logits{sfx}"] = p["query_logits"][0].detach().numpy()
        for i, aux in enumerate(p["aux_outputs"]):
            arrays[f"aux{i}_query_logits{sfx}"] = aux["query_logits"][0].detach().numpy()


# ------------------------------------------------------------------------------------------------
# readers
# ------------------------------------------------------------------------------------------------
def check_rows(name, got_C, got_F, gold_C, gold_F_sub, step, tol=1e-3, check=True):
    """→ (sym, err): rows the coordinate sets differ in, feature error of the subsample rows (max-abs normalised)."""
    gk, rk = keys(got_C), keys(gold_C)
    order = torch.argsort(gk)
    gk, gF = gk[order], got_F.detach().cpu()[order]
    common = np.intersect1d(gk.numpy(), rk.numpy())
    sym = (len(gk) - len(common)) + (len(rk) - len(common))
    assert sym <= max(2, 0.001 * len(rk)), f"{name}: coordinate sets differ in {sym} of {len(rk)} rows"
    sub_keys = rk[::step]
    pos = torch.searchsorted(gk, sub_keys).clamp(max=len(gk) - 1)
    hit = gk[pos] == sub_keys
    ref = torch.as_tensor(gold_F_sub)[hit]
    got = gF[pos[hit]]
    rowerr = (got.double() - ref.double()).abs().max(1)[0] / ref.double().abs().max()
    if sym == 0:
        err = float(rowerr.max())
    else:
        # an argmax near-tie kept/dropped `sym` voxels differently from the CPU run: the 3x3x3 convs behind the output
        # make their spatial neighbours differ too, everything else must still agree → judge the 99th percentile
        err = float(torch.quantile(rowerr, 0.99))
    assert (not check) or err <= tol, f"{name}: feature error {err:.3e} > {tol} (sym={sym})"
    return sym, err


def check_summary(name, C, F, gold, tol=1e-3, sym_frac=1e-3, q=0.99):
    """→ (exact_set, err).  exact_set: count, key sum and key xor all equal (bit-exact coordinate parity)."""
    k = keys(C)
    order = torch.argsort(k)
    k, F = k[order], F.detach().float().cpu()[order]
    kn = k.numpy().astype(np.uint64)
    n_gold = int(gold[f"{name}_n"][0])
    exact = (len(kn) == n_gold and np.add.reduce(kn) == gold[f"{name}_ksum"][0]
             and np.bitwise_xor.reduce(kn) == gold[f"{name}_ksum"][1])
    assert abs(len(kn) - n_gold) <= max(2, sym_frac * n_gold), f"{name}: {len(kn)} rows, reference {n_gold}"
    sub_k = torch.as_tensor(gold[f"{name}_subK"].astype(np.int64))
    pos = torch.searchsorted(k, sub_k).clamp(max=len(k) - 1)
    hit = k[pos] == sub_k
    assert float(hit.float().mean()) >= 1.0 - 2 * sym_frac - 2.0 / max(len(sub_k), 1), f"{name}: {int((~hit).sum())} subsample rows missing"
    ref = torch.as_tensor(gold[f"{name}_subF"])[hit].double()
    amax = float(gold[f"{name}_Fsum"][2])
    rowerr = (F[pos[hit]].double() - ref).abs().max(1)[0] / amax
    if exact:
        err = float(rowerr.max())
        s_err = abs(float(F.double().sum()) - float(gold[f"{name}_Fsum"][0])) / float(gold[f"{name}_Fsum"][1])
        assert s_err <= tol, f"{name}: checksum Σ differs by {s_err:.2e} of Σ|.|"
    else:       # an argmax / rank near-tie kept a few other voxels than the CPU run: neighbours differ, the rest must agree
        err = float(torch.quantile(rowerr, q))
        med = float(rowerr.median())
        assert med <= tol / 2, f"{name}: median feature error {med:.3e} > {tol / 2} (exact_set={exact})"
    assert err <= tol, f"{name}: feature error {err:.3e} > {tol} (exact_set={exact})"
    return exact, err


def logit_error(got, ref):
    """Max-abs error of dense logits, relative to the largest reference magnitude."""
    got, ref = torch.as_tensor(got).detach().double().cpu(), torch.as_tensor(ref).double()
    return float((got - ref).abs().max() / ref.abs().max())


def check_outputs(out, gold, meta, tol=1e-3, sym_frac=1e-3, q=0.99, head_tol=None, sem=True, aux=True, sums=False,
                  vox_step=None, worst=False):
    """Every output of the meta["n_infers"] subnets against a fixture of either format → {output: error report}.

    head_tol  bound of the voxel, query and aux logits (default tol; summary format: 5 tol for the query logits when the
              voxel set they attend over is not bit-identical to the reference's — a flipped voxel changes every query)
    sem       check the semantic logits; aux: check the aux query logits
    sums      rows format: when the voxel coordinate set is exact, also bound the checksums over all of its rows
    vox_step  rows format: row step of the voxel features when it differs from meta["row_step"]
    worst     rows format: bound only the worst error over all outputs (coordinate set differences still assert)"""
    fmt_rows = "vox_C" in gold or "vox_m0_C" in gold
    M, step = meta["n_infers"], meta["row_step"]
    head = head_tol or tol
    rep = {}
    for m in range(M):
        sfx = _sfx(m, M)
        p = out["panop_predictions"][m]
        sparse = [(f"sem{s}{sfx}", out["sem_logits_at_scales"][s][m], tol, step) for s in ((4, 2, 1) if sem else ())]
        sparse.append((f"vox{sfx}", p["voxel_logits"], head, vox_step or step))
        for name, st, t, stp in sparse:
            if fmt_rows:
                rep[name] = check_rows(name, st.C, st.F, gold[f"{name}_C"], gold[f"{name}_F"], stp, t, check=not worst)
            else:
                rep[name] = check_summary(name, st.C, st.F, gold, t, sym_frac, q)
        if sums and rep[f"vox{sfx}"][0] == 0:          # same coordinates: the checksums over all rows agree too
            f = p["voxel_logits"].F.detach().double()
            got = torch.stack([f.sum(), f.abs().sum()]).cpu().numpy()
            rep[f"vox_sum{sfx}"] = float(np.abs(got - gold[f"vox{sfx}_sum"]).max() / gold[f"vox{sfx}_sum"][1])
            assert rep[f"vox_sum{sfx}"] <= tol, rep
        rep[f"query{sfx}"] = logit_error(p["query_logits"][0], gold[f"query_logits{sfx}"])
        qtol = head_tol or (tol if fmt_rows or rep[f"vox{sfx}"][0] else 5 * tol)
        assert worst or rep[f"query{sfx}"] <= qtol, rep
        for i, a in enumerate(p["aux_outputs"] if aux else ()):
            rep[f"aux{i}{sfx}"] = logit_error(a["query_logits"][0], gold[f"aux{i}_query_logits{sfx}"])
            assert worst or rep[f"aux{i}{sfx}"] <= head, (i, sfx, rep[f"aux{i}{sfx}"])
    if worst:
        assert max(v[1] if isinstance(v, tuple) else v for v in rep.values()) <= tol, rep
    return rep


# ------------------------------------------------------------------------------------------------
# setup
# ------------------------------------------------------------------------------------------------
def manifest(name):
    return json.load(open(os.path.join(HERE, name)))


def fixture(name):
    z = np.load(os.path.join(HERE, name))
    return {k: z[k] for k in z.files}


def pasconet(M=1, f=64, num_queries=100, heavy=False, n_classes=20, in_channels=283, recipe=False):
    """PascoNet built under seed 0; recipe: with the name-seeded weights of recipe.py."""
    from pasco_b200.net3d import PascoNet
    torch.manual_seed(0)
    net = PascoNet(n_classes=n_classes, n_infers=M, in_channels=in_channels, f=f, num_queries=num_queries,
                   heavy_decoder=heavy)
    if recipe:
        from recipe import fill_state_dict
        net.load_reference_state_dict(fill_state_dict(net.reference_state_dict()))
    return net


INFER_MANIFEST = manifest("net_cfg1_infer_manifest.json")
STAT_SUFFIXES = (".running_mean", ".running_var")


def load_eval(net, tag, ref_names=True):
    """Recipe weights + the calibrated running statistics of eval fixture `tag`; eval mode, on the GPU → (net, gold).
    ref_names: `net` is a PascoNet (reference names through load_reference_state_dict), else the reference's Net."""
    from recipe import fill_state_dict
    gold = fixture(f"net_cfg1_infer_{tag}.npz")
    sd = fill_state_dict(net.reference_state_dict() if ref_names else net.state_dict())
    n = 0
    for k in sd:
        if k.endswith(STAT_SUFFIXES) and f"stat::{k}" in gold:
            sd[k] = torch.from_numpy(gold[f"stat::{k}"]).to(sd[k].dtype)
            n += 1
    assert n == len(INFER_MANIFEST["cases"][tag]["running_stats"]), (n, tag)
    (net.load_reference_state_dict if ref_names else net.load_state_dict)(sd)
    return net.cuda().eval(), gold


def scene(meta, M=1, dev="cuda"):
    """The fixture's synthetic scene, with the point features, coordinates and labels on `dev`."""
    from pasco_b200.synthetic import make_scene
    b = make_scene(meta["grid"], meta["occ"], M, in_ch=meta.get("in_channels", 283), n_classes=meta.get("n_classes", 20),
                   seed=meta["seed"])
    d = lambda t: t.to(dev)  # noqa: E731
    return dict(b, in_feats=[d(t) for t in b["in_feats"]], in_coords=[d(t) for t in b["in_coords"]],
                sem_labels={k: d(v) for k, v in b["sem_labels"].items()}, mask_classes=d(b["mask_classes"]))


def forward(net, sc, test=False):
    return net(sc["in_feats"], sc["in_coords"], sc["global_min_Cs"], sc["global_max_Cs"], sc["min_Cs"], sc["max_Cs"],
               test=test)


@contextlib.contextmanager
def launches():
    """(kind, path, Cin, Cout) of every convolution launch inside the block."""
    from pasco_b200 import ops
    got = []
    ops.PROFILE = []
    try:
        yield got
    finally:
        torch.cuda.synchronize()
        got.extend((kind, m["path"], m["Cin"], m["Cout"]) for kind, _, _, m in ops.PROFILE)
        ops.PROFILE = None
        ops.PAIR_COUNTS.clear()


def reference_net(n_infers=1, heavy=False, n_classes=20, in_channels=283, num_queries=100):
    """→ (MinkowskiEngine, the unmodified reference Net): `import MinkowskiEngine` resolves to compat/ → pasco_b200.me."""
    for p in (REF, os.path.join(ROOT, "compat")):
        if p not in sys.path:
            sys.path.insert(0, p)
    import MinkowskiEngine as ME
    assert "pasco_b200" in ME.__name__ or "compat" in (ME.__file__ or ""), f"MinkowskiEngine resolved to {ME.__file__}"
    assert ME.SparseTensor.__module__.startswith("pasco_b200.me"), ME.SparseTensor.__module__
    from pasco.models.net_panoptic_sparse import Net
    assert os.path.realpath(sys.modules["pasco.models.net_panoptic_sparse"].__file__).startswith(os.path.realpath(REF))
    freqs = {f"1_{s}": np.ones(n_classes) for s in (1, 2, 4)}
    torch.manual_seed(0)
    net = Net(n_classes=n_classes, class_names=[str(i) for i in range(n_classes)], class_weights=torch.ones(n_classes),
              encoder_dropouts=[0.0] * 3, decoder_dropouts=[0.0] * 3, dense3d_dropout=0.0, n_infers=n_infers,
              class_frequencies=freqs, in_channels=in_channels, num_queries=num_queries, f=64, heavy_decoder=heavy)
    return ME, net


def forward_reference(ME, net, b, dev, test=False):
    """What Net.step does up to the losses (net_panoptic_sparse.py:314-352), on device tensors."""
    d = lambda t: t.to(dev)  # noqa: E731
    in_coords, in_feats = net.feat([d(t) for t in b["in_feats"]], [d(t) for t in b["in_coords"]])
    x = net.augmenter.merge(ME.SparseTensor(in_feats, in_coords.int()))
    return net(x, 1, {k: d(v) for k, v in b["sem_labels"].items()}, global_min_coords=d(b["global_min_Cs"]),
               global_max_coords=d(b["global_max_Cs"]), min_Cs=[d(t) for t in b["min_Cs"]], max_Cs=[d(t) for t in b["max_Cs"]],
               Ts=[d(t) for t in b["Ts"]], is_predict_panop=True, return_ensemble=False, test=test)


# ------------------------------------------------------------------------------------------------
# kernel cases against the CPU oracle
# ------------------------------------------------------------------------------------------------
def engine():
    """pasco_b200.me over a freshly built library."""
    from pasco_b200 import build
    build.build()
    from pasco_b200 import me
    return me


def relerr(a, b):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    return float((a - b).abs().max() / b.abs().max().clamp(min=1e-30))


def sparse_scene(shape=(24, 20, 12), p=0.3, C=64, batch=1, lo=(0, 0, 0), seed=0, stride=1):
    """Batched Bernoulli coordinates (scaled by `stride`, shifted by `lo`) and random features."""
    import me_oracle as OR
    g = torch.Generator().manual_seed(seed)
    cs = []
    for b in range(batch):
        occ = torch.rand(*shape, generator=g) < p
        c = torch.nonzero(occ).int() * stride + torch.tensor(lo, dtype=torch.int32)
        cs.append(c)
    bc = OR.utils.batched_coordinates(cs)
    f = torch.randn(bc.shape[0], C, generator=g)
    return bc, f


def canon(C, F=None):
    """Sort rows by packed coordinate key."""
    C = C.detach().cpu()
    order = torch.argsort(keys(C))
    return (C[order], None if F is None else F.detach().cpu()[order])


def assert_same_sparse(got, ref, tol):
    gc, gf = canon(got.C, got.F)
    rc, rf = canon(ref.C, ref.F)
    assert gc.shape == rc.shape and torch.equal(gc, rc), "coordinate sets differ"
    assert got.tensor_stride == ref.tensor_stride
    e = relerr(gf, rf)
    assert e <= tol, f"feature error {e:.3e} > {tol}"
    return e


def conv_pair(ME, kind, cin, cout, seed=0, bias=False):
    import me_oracle as OR
    torch.manual_seed(seed)
    if kind == "k3":
        r = OR.MinkowskiConvolution(cin, cout, kernel_size=3, bias=bias, dimension=3)
        g = ME.MinkowskiConvolution(cin, cout, kernel_size=3, bias=bias, dimension=3)
    elif kind == "down":
        r = OR.MinkowskiConvolution(cin, cout, kernel_size=2, stride=2, dimension=3)
        g = ME.MinkowskiConvolution(cin, cout, kernel_size=2, stride=2, dimension=3)
    else:
        r = OR.MinkowskiConvolutionTranspose(cin, cout, kernel_size=2, stride=2, dimension=3, expand_coordinates=True)
        g = ME.MinkowskiConvolutionTranspose(cin, cout, kernel_size=2, stride=2, dimension=3, expand_coordinates=True)
    g.load_state_dict(r.state_dict())
    return r, g.cuda()


def run_conv_case(ME, kind, cin, cout, tol, shape=(20, 18, 10), p=0.3, bias=False):
    """One convolution ("k3", "down" or "up") forward + input and weight gradient on the engine `ME` against the oracle
    → (fwd, dgrad, wgrad) errors, each asserted <= tol."""
    import me_oracle as OR
    ts = 2 if kind == "up" else 1
    C, F = sparse_scene(shape=shape, p=p, C=cin, batch=2, lo=(-8, 0, 4), stride=ts)
    rconv, gconv = conv_pair(ME, kind, cin, cout, bias=bias)
    Fr = F.clone().requires_grad_(True)
    Fg = F.clone().cuda().requires_grad_(True)
    ref = rconv(OR.SparseTensor(Fr, C, tensor_stride=ts))
    got = gconv(ME.SparseTensor(Fg, C.cuda(), tensor_stride=ts))
    e_f = assert_same_sparse(got, ref, tol)
    # same upstream gradient on matching rows
    order_r = torch.argsort(keys(ref.C))
    order_g = torch.argsort(keys(got.C))
    gup = torch.randn(ref.F.shape, generator=torch.Generator().manual_seed(7))
    gr = torch.empty_like(gup)
    gr[order_r] = gup
    gg = torch.empty_like(gup)
    gg[order_g] = gup
    ref.F.backward(gr)
    got.F.backward(gg.cuda())
    e_i = relerr(Fg.grad, Fr.grad)
    e_w = relerr(gconv.kernel.grad, rconv.kernel.grad)
    assert e_i <= tol, f"dgrad error {e_i:.3e}"
    assert e_w <= tol, f"wgrad error {e_w:.3e}"
    if bias:
        assert relerr(gconv.bias.grad, rconv.bias.grad) <= tol
    return e_f, e_i, e_w
