"""Pins pasco_b200.net3d (the engine-native restatement of PaSCo's hot path) against golden vectors
produced by the UNMODIFIED reference running on the CPU oracle (tests/golden/make_golden.py).

CPU part : parameter names / shapes equal the reference's state_dict manifest (checkpoint drop-in).
GPU part : same recipe weights + same synthetic scene → sem logits at 3 scales, query logits and mask
           logits agree with the golden subsample within the north_star tolerance (1e-3, max-abs
           normalised).  Coordinate sets must be identical up to argmax near-ties (≤ 0.1 % of rows).
"""
import os
import sys

import numpy as np
import pytest
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import parity  # noqa: E402
from recipe import fill_state_dict  # noqa: E402

MANIFEST = parity.manifest("net_cfg1_manifest.json")


def test_state_dict_names_and_shapes_match_the_reference():
    sd = parity.pasconet().reference_state_dict()
    mine = {k: list(v.shape) for k, v in sd.items()}
    ref = MANIFEST["params"]
    assert sorted(mine) == sorted(ref), (sorted(set(ref) - set(mine))[:5], sorted(set(mine) - set(ref))[:5])
    bad = [k for k in ref if mine[k] != ref[k]]
    assert not bad, bad[:5]
    assert sum(int(np.prod(s)) for s in ref.values()) > 100e6


@pytest.mark.parametrize("variant,M,heavy", [("m2_light", 2, False), ("m1_heavy", 1, True), ("m3_light", 3, False)])
def test_state_dict_matches_reference_for_mimo_and_heavy_decoder(variant, M, heavy):
    """Checkpoint compatibility of the other shipped configurations: MIMO M=2/3 and heavy_decoder=True
    (manifests dumped from the reference's own Net.state_dict(), tests/golden/manifests_variants.json)."""
    ref = parity.manifest("manifests_variants.json")[variant]
    mine = {k: list(v.shape) for k, v in parity.pasconet(M, heavy=heavy).reference_state_dict().items()}
    assert sorted(mine) == sorted(ref), (sorted(set(ref) - set(mine))[:5], sorted(set(mine) - set(ref))[:5])
    assert all(mine[k] == ref[k] for k in ref)


def test_reference_state_dict_round_trip():
    net = parity.pasconet()
    sd = fill_state_dict(net.reference_state_dict())
    net.load_reference_state_dict(sd)
    back = net.reference_state_dict()
    assert all(torch.equal(back[k], sd[k]) for k in sd)
    with pytest.raises(KeyError):
        net.load_reference_state_dict({k: v for k, v in sd.items() if "enc_in_feats" not in k})


@pytest.mark.gpu
def test_full_forward_matches_reference_golden():
    from pasco_b200 import ops
    ops.set_precision("fp32")
    net = parity.pasconet(recipe=True).cuda().train()
    with torch.no_grad():
        out = parity.forward(net, parity.scene(MANIFEST))
    print("golden parity:", parity.check_outputs(out, parity.fixture("net_cfg1.npz"), MANIFEST))


@pytest.mark.gpu
def test_mimo_m2_forward_matches_reference_golden():
    """MIMO wrapper, M=2 (two scenes channel-concatenated through one trunk, per-subnet heads and transformer
    passes incl. the reference's zero-padding of the shorter subnet): golden from the unmodified reference."""
    from pasco_b200 import ops
    ops.set_precision("fp32")
    man = parity.manifest("net_cfg1_m2_manifest.json")
    net = parity.pasconet(2, recipe=True).cuda().train()
    with torch.no_grad():
        out = parity.forward(net, parity.scene(man, 2))
    print("MIMO M=2 golden parity:", parity.check_outputs(out, parity.fixture("net_cfg1_m2.npz"), man, worst=True))
