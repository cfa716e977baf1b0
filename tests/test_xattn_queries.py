"""Masked cross-attention beyond one 128-row query block (xattn.cu query blocks), from the kernel up to the network.

GPU part : the kernels against an fp64 reference for Q = 129 … 385, the rows of one query block independent of the
           others, two identical calls bit-identical, and PascoNet / the hooked unmodified reference with
           num_queries=200 against golden vectors the unmodified reference produced on the CPU oracle
           (tests/golden/make_golden_queries.py; coordinates and semantic logits do not depend on the query count and
           come from net_cfg1.npz).
CPU part : the golden manifest's parameter names / shapes equal PascoNet(num_queries=200).reference_state_dict().
"""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from recipe import fill_state_dict  # noqa: E402

NQ = 200
MANIFEST = parity.manifest(f"net_cfg1_q{NQ}_manifest.json")


def test_q200_manifest_matches_pasconet_state_dict():
    mine = {k: list(v.shape) for k, v in parity.pasconet(num_queries=NQ).reference_state_dict().items()}
    ref = MANIFEST["params"]
    assert MANIFEST["num_queries"] == NQ
    assert sorted(mine) == sorted(ref), (sorted(set(ref) - set(mine))[:5], sorted(set(mine) - set(ref))[:5])
    bad = [k for k in ref if mine[k] != ref[k]]
    assert not bad, bad[:5]
    assert ref["transformer_predictor.query_feat.weight"] == [NQ, 384]


# ------------------------------------------------------------------------------------------------
# kernel
# ------------------------------------------------------------------------------------------------
def _inputs(Q, P, H, D, masked, seed):
    g = torch.Generator().manual_seed(seed)
    q, k, v = (torch.randn(n, H * D, generator=g) for n in (Q, P, P))
    mask = None
    if masked:
        mask = torch.rand(Q, P, generator=g) < 0.6
        for r, key in ((min(128 + 5, Q - 1), P // 2), (Q - 1, P - 1)):   # a single visible key in the 2nd / last block
            mask[r] = True
            mask[r, key] = False
        mask[mask.all(1)] = False
    up = torch.randn(Q, H * D, generator=g)
    return q, k, v, mask, up


def _run(q, k, v, mask, up, H):
    """forward + backward on the GPU → out, lse, dq, dk, dv"""
    import ctypes as C
    from pasco_b200 import ops
    from pasco_b200._lib import ptr
    Q, HD = q.shape
    P, D = k.shape[0], HD // H
    qg, kg, vg = (t.cuda().contiguous() for t in (q, k, v))
    bits = ops.pack_mask_bits(mask.cuda()) if mask is not None else None
    out = torch.zeros(Q, HD, device="cuda")
    lse = torch.empty(H, Q, device="cuda")
    ops.call("pasco_xattn_forward", ptr(qg), ptr(kg), ptr(vg), ptr(bits), Q, P, H, D, C.c_float(D ** -0.5), ptr(out),
             ptr(lse))
    dq, dk, dv = torch.zeros_like(qg), torch.empty_like(kg), torch.empty_like(vg)
    go = up.cuda().contiguous()
    ops.call("pasco_xattn_backward", ptr(qg), ptr(kg), ptr(vg), ptr(bits), ptr(lse), ptr(out), ptr(go), Q, P, H, D,
             C.c_float(D ** -0.5), ptr(dq), ptr(dk), ptr(dv))
    torch.cuda.synchronize()
    return out, lse, dq, dk, dv


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [True, False])
@pytest.mark.parametrize("H,D", [(8, 48), (6, 64), (4, 20)])
@pytest.mark.parametrize("P", [37, 3000, 20011])
@pytest.mark.parametrize("Q", [129, 150, 200, 256, 385])
def test_xattn_many_queries_matches_fp64_reference(Q, P, H, D, masked):
    from pasco_b200 import ops
    q, k, v, mask, up = _inputs(Q, P, H, D, masked, seed=Q * 100003 + P)

    def ref(q, k, v):
        hv = lambda t: t.view(t.shape[0], H, D).transpose(0, 1)              # noqa: E731
        s = torch.bmm(hv(q) * D ** -0.5, hv(k).transpose(1, 2))
        if mask is not None:
            s = s.masked_fill(mask.cuda().unsqueeze(0), float("-inf"))
        return torch.bmm(torch.softmax(s, -1), hv(v)).transpose(0, 1).reshape(Q, H * D)

    qr, kr, vr = (t.cuda().double().requires_grad_(True) for t in (q, k, v))   # fp64 on the device: Q x P x H is large
    yr = ref(qr, kr, vr)
    (yr * up.cuda().double()).sum().backward()
    qg, kg, vg = (t.clone().cuda().requires_grad_(True) for t in (q, k, v))
    yg = ops.MaskedCrossAttention.apply(qg, kg, vg, mask.cuda() if mask is not None else None, H)
    (yg * up.cuda()).sum().backward()
    e = parity.relerr(yg, yr)
    eg = max(parity.relerr(qg.grad, qr.grad), parity.relerr(kg.grad, kr.grad), parity.relerr(vg.grad, vr.grad))
    print(f"xattn Q={Q} P={P} H={H} D={D} masked={masked}: fwd {e:.2e} grads {eg:.2e}")
    assert e <= 1e-4 and eg <= 5e-4


def _chunks(P, H, nqb):
    """xattn.cu pick_chunks: key chunks per (query block, head), about one CTA per SM."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    return max(1, min((P + 63) // 64, -(-sms // (H * nqb))))


@pytest.mark.gpu
@pytest.mark.parametrize("masked", [True, False])
def test_xattn_query_blocks_are_independent(masked):
    """A query row's result depends on its own query only: rows 0..127 of a Q = 200 call equal a Q = 128 call on the
    first 128 queries bit-for-bit when both split the keys into the same chunks, and rows 0..199 of a Q = 200 call
    equal those of a Q = 256 call (same query blocks and chunks) bit-for-bit at a full-size key count."""
    H, D = 8, 48
    P_small = 64 * _chunks(10 ** 9, H, 2)                  # as many key tiles as chunks: both calls use one tile each
    assert _chunks(P_small, H, 1) == _chunks(P_small, H, 2)
    q, k, v, mask, _ = _inputs(256, P_small, H, D, masked, seed=7)
    o200, l200, *_ = _run(q[:200], k, v, mask[:200] if masked else None, torch.zeros(200, H * D), H)
    o128, l128, *_ = _run(q[:128], k, v, mask[:128] if masked else None, torch.zeros(128, H * D), H)
    assert torch.equal(o200[:128], o128) and torch.equal(l200[:, :128], l128)

    q, k, v, mask, up = _inputs(256, 20011, H, D, masked, seed=8)
    o200, l200, dq200, *_ = _run(q[:200], k, v, mask[:200] if masked else None, up[:200], H)
    o256, l256, dq256, *_ = _run(q, k, v, mask, torch.cat([up[:200], torch.zeros(56, H * D)]), H)
    assert torch.equal(o200, o256[:200]) and torch.equal(l200, l256[:, :200]) and torch.equal(dq200, dq256[:200])


@pytest.mark.gpu
def test_xattn_many_queries_is_deterministic():
    H, D = 8, 48
    q, k, v, mask, up = _inputs(200, 20011, H, D, True, seed=9)
    a = _run(q, k, v, mask, up, H)
    b = _run(q, k, v, mask, up, H)
    for name, x, y in zip(("out", "lse", "dq", "dk", "dv"), a, b):
        assert torch.equal(x, y), name


# ------------------------------------------------------------------------------------------------
# network: PascoNet and the hooked unmodified reference with num_queries=200
# ------------------------------------------------------------------------------------------------
def _check_against_gold(out, sem=True):
    """Coordinates and semantic logits from net_cfg1 at its row step, the voxel rows at the q200 step."""
    p = out["panop_predictions"][0]
    assert p["query_logits"].shape[-2] == NQ and p["voxel_logits"].F.shape[1] == NQ
    gold = dict(parity.fixture(MANIFEST["coords_and_sem_from"]), **parity.fixture(f"net_cfg1_q{NQ}.npz"))
    return parity.check_outputs(out, gold, parity.manifest("net_cfg1_manifest.json"), sem=sem, sums=True,
                                vox_step=MANIFEST["row_step"])


@pytest.mark.gpu
def test_pasconet_200_queries_matches_reference_golden_and_trains():
    from pasco_b200 import ops
    from pasco_b200.losses import total_loss
    ops.set_precision("fp32")
    net = parity.pasconet(num_queries=NQ, recipe=True).cuda().train()
    sc = parity.scene(MANIFEST)
    with torch.no_grad():
        out = parity.forward(net, sc)
    print("PascoNet num_queries=200 vs golden:", _check_against_gold(out))

    # one training step: forward + loss + backward, every transformer parameter gets a finite gradient
    opt = torch.optim.SGD(net.parameters(), lr=1e-4)
    loss = total_loss(parity.forward(net, sc), sc, 20, net.class_frequencies)
    loss.backward()
    torch.cuda.synchronize()
    assert torch.isfinite(loss), loss
    tp = [(n, p) for n, p in net.named_parameters() if n.startswith("transformer_predictor.")]
    assert len(tp) > 50, len(tp)
    missing = [n for n, p in tp if p.grad is None]
    bad = [n for n, p in tp if p.grad is not None and not torch.isfinite(p.grad).all()]
    assert not missing and not bad, (missing[:5], bad[:5])
    assert float(net.transformer_predictor.query_feat.weight.grad[128:].abs().max()) > 0   # the second query block
    opt.step()


@pytest.mark.gpu
@pytest.mark.skipif(not os.path.isdir(os.path.join(parity.REF, "pasco")),
                    reason="no upstream PaSCo checkout was readable when build() ran: oracle/_ref not staged")
def test_reference_200_queries_with_attention_hooks_matches_golden():
    from pasco_b200 import ops, hooks
    ops.set_precision("fp32")
    dev = torch.device("cuda")
    ME, net = parity.reference_net(num_queries=NQ)
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.to(dev).train()
    assert hooks.install()
    try:
        calls0 = ops.CALLS
        out = parity.forward_reference(ME, net, parity.scene(MANIFEST), dev)
        assert ops.CALLS - calls0 > 100
        report = _check_against_gold(out, sem=False)
        p = out["panop_predictions"][0]
        (p["voxel_logits"].F.square().mean() + p["query_logits"].square().mean()).backward()
        g = net.transformer_predictor.transformer_cross_attention_layers[1].multihead_attn.in_proj_weight.grad
        assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0
        print("drop-in with attention hooks, num_queries=200, vs golden:", report)
    finally:
        hooks.uninstall()
