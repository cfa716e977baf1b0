"""The real drop-in: the UNMODIFIED reference model (`pasco.models.net_panoptic_sparse.Net`, staged by build() through
oracle/stage_reference.py under oracle/_ref/, never committed) runs on the GPU
with `import MinkowskiEngine` / `torch_scatter` resolving to compat/ → pasco_b200.me → libpasco_sm100.so, and its
outputs are compared (a) with the golden vectors the same reference produced on the CPU oracle and (b) with the
engine-native PascoNet on the same weights and scene.

Reference path exercised: net_panoptic_sparse.py:210-312 → unet3d_sparse_v2.py:216-256 (encoder_v2, dense bottleneck
through nn.Conv3d, decoder_v3 incl. predict_completion_sem_logit / predict_panop, transformer_predictor_v2).
Skips cleanly when oracle/_ref is absent (no upstream checkout at build time).
"""
import os
import sys

import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from recipe import fill_state_dict  # noqa: E402

MANIFEST = parity.manifest("net_cfg1_manifest.json")
pytestmark = [pytest.mark.gpu,
              pytest.mark.skipif(not os.path.isdir(os.path.join(parity.REF, "pasco")), reason="no upstream PaSCo checkout was readable when build() ran: oracle/_ref not staged")]


def test_unmodified_reference_net_on_the_engine_matches_golden_and_pasconet():
    from pasco_b200 import ops
    ops.set_precision("fp32")
    dev = torch.device("cuda")
    ME, net = parity.reference_net()
    sd = fill_state_dict(net.state_dict())
    net.load_state_dict(sd)
    net.to(dev).train()
    sc = parity.scene(MANIFEST)
    calls0 = ops.CALLS
    with torch.no_grad():
        out = parity.forward_reference(ME, net, sc, dev)
    assert ops.CALLS - calls0 > 100, "the reference forward did not run on the engine's C-ABI"
    report = parity.check_outputs(out, parity.fixture("net_cfg1.npz"), MANIFEST)
    print("drop-in (unmodified reference on pasco_b200.me) vs golden:", report)

    # (b) the engine-native composition on the same weights and scene agrees with the reference-driven one
    mine = parity.pasconet()
    mine.load_reference_state_dict({k: v for k, v in sd.items()})
    mine.to(dev).train()
    with torch.no_grad():
        o2 = parity.forward(mine, sc)
    step = MANIFEST["row_step"]
    for s in (4, 2, 1):
        a, c = out["sem_logits_at_scales"][s][0], o2["sem_logits_at_scales"][s][0]
        order = torch.argsort(parity.keys(a.C))
        sym, err = parity.check_rows(f"native-vs-dropin sem{s}", c.C, c.F, a.C.cpu()[order].numpy(),
                                     a.F.detach().cpu()[order][::step].numpy(), step)
        assert err <= 1e-3


def test_reference_with_attention_hooks_matches_golden():
    """pasco_b200.hooks.install(): the unmodified reference's CrossAttentionLayer / compute_attn_mask run on the xattn
    kernels and the sparse mask instead of nn.MultiheadAttention and the dense [100, X, Y, Z] volume — same golden."""
    from pasco_b200 import ops, hooks
    ops.set_precision("fp32")
    dev = torch.device("cuda")
    ME, net = parity.reference_net()
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.to(dev).train()
    assert hooks.install()
    try:
        out = parity.forward_reference(ME, net, parity.scene(MANIFEST), dev)
        p = out["panop_predictions"][0]
        report = parity.check_outputs(out, parity.fixture("net_cfg1.npz"), MANIFEST, sem=False)
        (p["voxel_logits"].F.square().mean() + p["query_logits"].square().mean()).backward()
        g = net.transformer_predictor.transformer_cross_attention_layers[1].multihead_attn.in_proj_weight.grad
        assert g is not None and torch.isfinite(g).all() and float(g.abs().max()) > 0
        print("drop-in with attention hooks vs golden:", report)
    finally:
        hooks.uninstall()


def test_unmodified_reference_training_step_backward_runs_on_the_engine():
    """fwd + bwd of the unmodified reference network (loss = Σ logits²) — every parameter on the path gets a finite
    gradient through the engine's autograd Functions."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    dev = torch.device("cuda")
    ME, net = parity.reference_net()
    net.load_state_dict(fill_state_dict(net.state_dict()))
    net.to(dev).train()
    out = parity.forward_reference(ME, net, parity.scene(MANIFEST), dev)
    loss = sum(lg.F.square().mean() for s in (4, 2, 1) for lg in out["sem_logits_at_scales"][s])
    p = out["panop_predictions"][0]
    loss = loss + p["voxel_logits"].F.square().mean() + p["query_logits"].square().mean()
    loss.backward()
    torch.cuda.synchronize()
    named = [(n, q) for n, q in net.named_parameters() if q.grad is not None]
    assert len(named) > 300, len(named)
    bad = [n for n, q in named if not torch.isfinite(q.grad).all()]
    assert not bad, bad[:5]
    for must in ("unet3d.encoder.s1s2.0.net.0.kernel", "unet3d.dense3d.0.a_conv4.0.weight",
                 "unet3d.decoder_generative.voxel_feats.scale1_infer0.0.kernel", "transformer_predictor.input_projs.2.weight"):
        g = dict(named).get(must)
        assert g is not None and float(g.grad.abs().max()) > 0, must
