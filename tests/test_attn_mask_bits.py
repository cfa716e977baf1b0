"""The cross-attention mask as bit rows built on the device (ops.attention_mask_bits, csrc/attn_mask.cu), and the
unmodified reference's TransformerPredictorV2.forward running on them through hooks.install().

CPU: `oracle_bits`, a torch restatement of the bit semantics, against the reference's own definition of the mask
(transformer_predictor_v2.py:220-289 and 164: a dense volume of the thresholded logits max-pooled to the key scale,
read at the key voxels, all-masked rows cleared), written out per voxel in Python.
GPU: the kernel against that oracle and against the [Q, P] bool path it replaces; the hooked reference against the
golden vectors and the hooks-off reference; the memory the hooked forward's mask path adds at 1 M keys."""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from recipe import fill_state_dict  # noqa: E402

needs_ref = pytest.mark.skipif(not os.path.isdir(os.path.join(parity.REF, "pasco")),
                               reason="no upstream PaSCo checkout was readable when build() ran: oracle/_ref not staged")


def pack(mask: torch.Tensor) -> torch.Tensor:
    """bool [Q, P] (True = masked) → int32 [Q, 2*ceil(P/64)], keys beyond P masked (ops.pack_mask_bits' layout)."""
    from pasco_b200 import ops
    return ops.pack_mask_bits(mask)


def oracle_bits(logits, key_parent, rows=None, parent_of=None, n_parent=None):
    """ops.attention_mask_bits restated in torch (any device): the same arguments, the same words."""
    keep = logits > 0
    if rows is not None:
        keep = keep[rows.long()]
    if parent_of is not None:
        ok = parent_of >= 0
        pooled = torch.zeros(n_parent, keep.shape[1], dtype=torch.int32, device=keep.device)
        pooled = pooled.index_add_(0, parent_of[ok].long(), keep[ok].int()) > 0
    else:
        pooled = keep
    kp = key_parent.long()
    at = pooled[kp.clamp(min=0)] & (kp >= 0)[:, None]
    m = ~at.t()
    return pack(m & ~m.all(1, keepdim=True))


def definition_bits(C1, logits, Cs, scale):
    """The reference's mask from coordinates, one voxel at a time: the first row of a voxel stands for it, a key is
    unmasked for q when some voxel of its stride-`scale` block has logit > 0, a query with every key masked attends to
    all of them.  C1 [P1, 3], Cs [P, 3] (x, y, z)."""
    Q = logits.shape[1]
    first = {}
    for r, c in enumerate(map(tuple, C1.tolist())):
        first.setdefault(c, r)
    block = {}
    for c, r in first.items():
        p = tuple((x // scale) * scale for x in c)
        block[p] = block.get(p, torch.zeros(Q, dtype=torch.bool)) | (logits[r] > 0)
    none = torch.zeros(Q, dtype=torch.bool)
    m = torch.stack([~block.get(tuple(c), none) for c in Cs.tolist()], 1)
    m[m.all(1)] = False
    return pack(m)


def case(Q, n_vox, n_pad, n_keys, n_orphans, scale, seed):
    """A MIMO-padded scene: n_vox voxels of a 20 x 16 x 8 box plus n_pad zero rows, logits [P1, Q] with an all-negative
    query (0), a query with one positive voxel (1) and sparse positives elsewhere; n_keys stride-`scale` keys drawn from
    the voxels' blocks (some whose voxels are all negative), n_orphans keys with no voxel and two zero (padding) keys.
    → (C1, logits, Cs, rows, parent_of, n_parent, key_parent) on the CPU, index maps as the coordinate manager makes."""
    g = torch.Generator().manual_seed(seed)
    box = torch.tensor([20, 16, 8])
    cells = torch.randperm(int(box.prod()), generator=g)[:n_vox]
    C1 = torch.stack([cells // 128, (cells // 8) % 16, cells % 8], 1)
    C1 = torch.cat([C1, torch.zeros(n_pad, 3, dtype=torch.long)])
    P1 = C1.shape[0]
    logits = torch.randn(P1, Q, generator=g) - 1.5
    logits[:, 0] = -torch.rand(P1, generator=g)
    logits[:, 1] = -1.0
    logits[int(torch.randint(P1, (1,), generator=g)), 1] = 0.5
    first, rows = {}, []
    for r, c in enumerate(map(tuple, C1.tolist())):
        if c not in first:
            first[c] = len(rows)
            rows.append(r)
    parents, parent_of = {}, []
    for c in first:
        p = tuple((x // scale) * scale for x in c)
        parent_of.append(parents.setdefault(p, len(parents)))
    plist = list(parents)
    pick = torch.randperm(len(plist), generator=g)[:min(n_keys, len(plist))].tolist()
    keys = [plist[i] for i in pick]
    keys += [(40 * scale + i * scale, 0, 0) for i in range(n_orphans)] + [(0, 0, 0)] * 2
    keys = [keys[i] for i in torch.randperm(len(keys), generator=g).tolist()]
    Cs = torch.tensor(keys, dtype=torch.long)
    key_parent = torch.tensor([parents.get(k, -1) for k in keys], dtype=torch.int32)
    i32 = lambda v: torch.tensor(v, dtype=torch.int32)  # noqa: E731
    rows_t = None if len(rows) == P1 else i32(rows)
    par_t = None if scale == 1 else i32(parent_of)
    return C1, logits, Cs, rows_t, par_t, len(parents), key_parent


CASES = [  # Q, voxels, padded rows, keys, keys with no voxel, scale, seed
    (100, 700, 37, 500, 0, 1, 0),
    (100, 700, 37, 301, 9, 2, 1),
    (7, 1500, 0, 190, 5, 4, 2),
    (200, 900, 12, 431, 3, 2, 3),
    (129, 1200, 64, 640, 0, 1, 4),
    (33, 400, 5, 63, 1, 4, 5),
]


# ------------------------------------------------------------------------------------------------
# CPU: the oracle against the reference's definition
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("Q,n_vox,n_pad,n_keys,n_orphans,scale,seed", CASES)
def test_oracle_matches_the_reference_definition(Q, n_vox, n_pad, n_keys, n_orphans, scale, seed):
    C1, logits, Cs, rows, parent_of, n_parent, key_parent = case(Q, n_vox, n_pad, n_keys, n_orphans, scale, seed)
    if scale == 1:
        n_parent = None
    got = oracle_bits(logits, key_parent, rows, parent_of, n_parent)
    want = definition_bits(C1, logits, Cs, scale)
    assert torch.equal(got, want)
    P = Cs.shape[0]
    assert got.shape == (Q, 2 * ((P + 63) // 64))
    m = ((got.long()[:, :, None] >> torch.arange(32)) & 1).bool().flatten(1)          # [Q, 32·W]
    assert m[:, P:].all(), "keys beyond P are masked"
    assert not m[0, :P].any(), "an all-masked query attends to every key"
    assert m[2:, :P].any(), "some keys are masked"
    if n_orphans:
        assert (key_parent < 0).any()


# ------------------------------------------------------------------------------------------------
# GPU: the kernel
# ------------------------------------------------------------------------------------------------
def _on(dev, *ts):
    return [t.to(dev) if torch.is_tensor(t) else t for t in ts]


@pytest.mark.gpu
@pytest.mark.parametrize("Q,n_vox,n_pad,n_keys,n_orphans,scale,seed", CASES)
def test_kernel_matches_oracle_and_is_deterministic(Q, n_vox, n_pad, n_keys, n_orphans, scale, seed):
    from pasco_b200 import ops
    _, logits, _, rows, parent_of, n_parent, key_parent = case(Q, n_vox, n_pad, n_keys, n_orphans, scale, seed)
    want = oracle_bits(logits, key_parent, rows, parent_of, n_parent)
    lg, kp, rw, po = _on("cuda", logits, key_parent, rows, parent_of)
    wide = torch.nn.functional.pad(lg, (0, 64 - Q % 64 if Q % 64 else 0))          # a column slice, as pred_heads gives
    got = ops.attention_mask_bits(wide[:, :Q], kp, rw, po, n_parent)
    again = ops.attention_mask_bits(lg, kp, rw, po, n_parent)
    torch.cuda.synchronize()
    assert torch.equal(got.cpu(), want) and torch.equal(got, again)


def _todays_bits(logits, mgr, key1, uidx, Cs, scale):
    """The bool path the bit builder replaces (MaskTransformer.attn_mask before): thresholded rows, max-pooled, looked
    up at the keys, a [Q, P] bool, packed."""
    from pasco_b200 import ops
    keep = (logits.detach() > 0).float()
    if uidx is not None:
        keep = ops._gather_rows(keep.contiguous(), uidx)
    if scale == 1:
        pooled, key_s = keep, key1
    else:
        key_s = mgr.stride(key1, scale)
        pooled = ops.MaxPoolRows.apply(keep, mgr.pool_map(key1, key_s, scale), mgr.size(key_s))
    at = ops._gather_rows(pooled.contiguous(), ops.hash_lookup(mgr._table(key_s), Cs))
    m = (at == 0).t().contiguous()
    return ops.pack_mask_bits(m & ~m.all(1, keepdim=True))


@pytest.mark.gpu
@pytest.mark.parametrize("scale", [1, 2, 4])
def test_kernel_matches_the_bool_path_on_random_padded_rows(scale):
    from pasco_b200 import me as ME, ops
    g = torch.Generator().manual_seed(scale)
    cells = torch.randperm(64 * 64 * 8, generator=g)[:9000]
    C1 = torch.stack([torch.zeros_like(cells), cells // 512, (cells // 8) % 64, cells % 8], 1).int()
    C1 = torch.cat([C1, torch.zeros(301, 4, dtype=torch.int32)]).cuda()                # MIMO padding rows
    logits = (torch.randn(C1.shape[0], 128, generator=g) - 1.0).cuda()[:, :100]
    mgr = ME.CoordinateManager()
    key1, uidx = mgr.insert_and_map(C1)
    assert uidx is not None
    key_s = mgr.stride(key1, scale)
    Cs = torch.cat([mgr.get_coordinates(key_s), torch.zeros(77, 4, dtype=torch.int32, device="cuda"),
                    torch.tensor([[0, 200, 0, 0], [0, 0, 300, 0]], dtype=torch.int32, device="cuda")])
    parent_of = None if scale == 1 else mgr.pool_map(key1, key_s, scale)
    got = ops.attention_mask_bits(logits, ops.hash_lookup(mgr._table(key_s), Cs), uidx, parent_of, mgr.size(key_s))
    assert torch.equal(got, _todays_bits(logits, mgr, key1, uidx, Cs, scale))


@pytest.mark.gpu
@pytest.mark.parametrize("M", [1, 2])
def test_pasconet_masks_match_the_bool_path_on_the_fixture_scene(M, monkeypatch):
    """Every level's mask of PascoNet's forward on the net_cfg1 (M = 1) / net_cfg1_m2 (M = 2, padded rows) scene equals
    the packed bool mask of the path it replaces, word for word."""
    from pasco_b200 import ops
    from pasco_b200.net3d import MaskTransformer
    ops.set_precision("fp32")
    man = parity.manifest("net_cfg1_manifest.json" if M == 1 else "net_cfg1_m2_manifest.json")
    net = parity.pasconet(M, recipe=True).cuda().train()
    seen = []
    build = MaskTransformer.attn_mask

    def checked(self, mask_logits, vox, vox_rows, src_C, scale):
        bits = build(self, mask_logits, vox, vox_rows, src_C, scale)
        want = _todays_bits(mask_logits, vox.coordinate_manager, vox.coordinate_map_key, vox_rows, src_C, scale)
        seen.append((scale, vox_rows is not None, torch.equal(bits, want)))
        return bits

    monkeypatch.setattr(MaskTransformer, "attn_mask", checked)
    with torch.no_grad():
        parity.forward(net, parity.scene(man, M))
    assert len(seen) == 3 * M and sorted({s for s, _, _ in seen}) == [1, 2, 4]
    assert all(ok for _, _, ok in seen), seen
    print(f"M={M}: (scale, padded rows, equal) per mask:", seen)


# ------------------------------------------------------------------------------------------------
# GPU: the unmodified reference through the forward hook
# ------------------------------------------------------------------------------------------------
def _reference(M):
    from pasco_b200 import ops
    ops.set_precision("fp32")
    ME, net = parity.reference_net(n_infers=M)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    return ME, net.cuda().train()


@pytest.mark.gpu
@needs_ref
@pytest.mark.parametrize("M", [1, 2])
def test_reference_forward_hook_matches_golden_hooks_off_and_trains(M):
    from pasco_b200 import hooks, ops
    man = parity.manifest("net_cfg1_manifest.json" if M == 1 else "net_cfg1_m2_manifest.json")
    ME, net = _reference(M)
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    sc = parity.scene(man, M)
    torch.manual_seed(0)                  # the reference's point voxeliser shuffles its points: the same draw both times
    off = parity.forward_reference(ME, net, sc, "cuda")
    assert hooks.install()
    try:
        assert TransformerPredictorV2.forward is hooks._transformer_forward
        torch.manual_seed(0)
        out = parity.forward_reference(ME, net, sc, "cuda")
        gold = parity.fixture("net_cfg1.npz" if M == 1 else "net_cfg1_m2.npz")
        report = parity.check_outputs(out, gold, man, sem=False, worst=M == 2)      # test_golden_net's M = 2 bound
        print(f"reference M={M} with the forward hook vs golden:", report)
        for m in range(M):
            a, b = out["panop_predictions"][m], off["panop_predictions"][m]
            assert torch.equal(a["voxel_logits"].C, b["voxel_logits"].C)
            errs = [parity.relerr(a["voxel_logits"].F, b["voxel_logits"].F),
                    parity.relerr(a["query_logits"], b["query_logits"])]
            errs += [parity.relerr(x["query_logits"], y["query_logits"])
                     for x, y in zip(a["aux_outputs"], b["aux_outputs"])]
            assert len(a["aux_outputs"]) == len(b["aux_outputs"]) == 3
            print(f"subnet {m}: hooks on vs off, voxel / query / aux logits:", ["%.2e" % e for e in errs])
            assert max(errs) <= 1e-3, errs
        loss = sum(p["voxel_logits"].F.square().mean() + p["query_logits"].square().mean()
                   for p in out["panop_predictions"])
        loss.backward()
        tp = net.transformer_predictor
        for i in range(3):
            g = tp.transformer_cross_attention_layers[i].multihead_attn.in_proj_weight.grad
            assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0, i
        assert float(tp.query_feat.weight.grad[(M - 1) * 100:].abs().max()) > 0     # the last subnet's queries
    finally:
        hooks.uninstall()
    assert TransformerPredictorV2.forward is TransformerPredictorV2._pasco_b200_orig_forward
    assert ops.CALLS > 0


@pytest.mark.gpu
@needs_ref
def test_hooked_forward_mask_memory_is_bounded_by_shapes(monkeypatch):
    """A transformer call of M = 2 subnets over P1 ≈ 1 M scale-1 keys (the second subnet zero-padded): each level's
    mask adds at most a bound computed from shapes — the bits, the pooled query words and the coordinate maps — far
    below the reference's [B·heads, Q, P] bool mask (let alone its int64 row sum)."""
    from pasco_b200 import hooks
    parity.reference_net()                                  # sys.path: `pasco` from oracle/_ref on pasco_b200.me
    from pasco.models.transformer.transformer_predictor_v2 import TransformerPredictorV2
    torch.manual_seed(0)
    B, Q, H, d, c = 2, 100, 8, 96, 16
    tp = TransformerPredictorV2(in_channels=[c, c, c], hidden_dim=d, num_queries=Q, nheads=H, dim_feedforward=128,
                                mask_dim=c, n_infers=B).cuda().eval()
    dev = torch.device("cuda")
    sizes = (1_000_000, 900_000)
    xs, keep_pad = {}, torch.zeros(B, sizes[0], dtype=torch.bool, device=dev)
    for s in (1, 2, 4):
        Fs, Cs = [], []
        for b, n in enumerate(sizes):
            g = torch.Generator(device=dev).manual_seed(b)
            cells = torch.randperm(256 * 256 * 32, device=dev, generator=g)[:n]
            C = torch.stack([torch.zeros_like(cells), cells // 8192, (cells // 32) % 256, cells % 32], 1).int()
            C = torch.unique(torch.div(C, s, rounding_mode="floor") * s, dim=0) if s > 1 else C
            Cs.append(C)
            if s == 1:
                keep_pad[b, :n] = True
        n_max = max(C.shape[0] for C in Cs)
        Cs = [torch.nn.functional.pad(C, (0, 0, 0, n_max - C.shape[0])) for C in Cs]
        xs[s] = (torch.randn(B, n_max, c, device=dev), torch.stack(Cs))
    P1 = xs[1][0].shape[1]
    assert xs[1][0].shape[1] == sizes[0]

    added = []
    mask_bits = hooks._mask_bits

    def measured(voxels, logits, src_C, scale):
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        bits = mask_bits(voxels, logits, src_C, scale)
        torch.cuda.synchronize()
        n1, P = voxels[0].size(voxels[1]), src_C.shape[0]
        QW, W = (Q + 31) // 32, 2 * ((P + 63) // 64)
        bound = 4 * Q * W + n1 * (4 * QW + 160) + 48 * P + (8 << 20)
        added.append((scale, torch.cuda.max_memory_allocated() - base, bound, P))
        return bits

    monkeypatch.setattr(hooks, "_mask_bits", measured)
    assert hooks.install()
    try:
        with torch.no_grad():
            torch.cuda.synchronize()
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
            out = tp(xs, (torch.empty(B, 1, 1, device=dev), None), None, None, keep_pad)
            torch.cuda.synchronize()
        forward_peak = torch.cuda.max_memory_allocated() - base
    finally:
        hooks.uninstall()
    assert len(out) == B and out[1]["voxel_logits"].F.shape == (sizes[1], Q)
    assert len(added) == 3 * B
    print(f"P1 = {P1}: forward peak added {forward_peak / 2**20:.0f} MiB; per mask (scale, MiB added, MiB bound):",
          [(s, round(a / 2**20), round(bd / 2**20)) for s, a, bd, _ in added])
    for s, a, bd, P in added:
        assert a <= bd, (s, a, bd)
        assert bd < B * H * Q * P1 / 4
