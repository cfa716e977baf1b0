"""PASCO_B200_HOOKS (pasco_b200/hooks.py):

  * its values: "" and "0" no group, "1" the attention group, else a comma list of group names; every group has
    trigger modules.
In a fresh interpreter each:
  * an unknown group name raises ValueError whichever of pasco_b200.hooks, pasco_b200.me or compat's MinkowskiEngine is
    imported first; unset, "1" and a valid list import cleanly in every order;
  * the requested groups install lazily: on the first SparseTensor construction after their trigger modules have been
    imported (needs oracle/_ref).
"""
import os
import subprocess
import sys

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
REF = os.path.join(ROOT, "oracle", "_ref")
PATHS = f"import sys; sys.path[:0] = [{ROOT!r}, {os.path.join(ROOT, 'compat')!r}, {REF!r}]\n"
FIRST = ("pasco_b200.hooks", "pasco_b200.me", "MinkowskiEngine")


def test_hook_switch_values():
    from pasco_b200.hooks import _GROUPS, _parse_groups
    assert _parse_groups("0") == frozenset() and _parse_groups("") == frozenset()
    assert _parse_groups("1") == {"attention"}
    for g in ("attention", "postprocess", "evaluate", "criterion", "trunk", "decoder", "transformer"):
        assert _parse_groups(g) == {g}
    assert _parse_groups(" trunk , criterion ") == {"trunk", "criterion"}
    assert _parse_groups(" decoder , trunk ") == {"decoder", "trunk"}
    assert _parse_groups(" attention , transformer ") == {"attention", "transformer"}
    assert _parse_groups("attention,postprocess") == {"attention", "postprocess"}
    assert _parse_groups("attention,postprocess,evaluate") == {"attention", "postprocess", "evaluate"}
    assert _parse_groups("attention,postprocess,evaluate,criterion") == {"attention", "postprocess", "evaluate",
                                                                         "criterion"}
    assert _parse_groups("attention,postprocess,evaluate,criterion,trunk") == {"attention", "postprocess", "evaluate",
                                                                               "criterion", "trunk"}
    assert _parse_groups("attention,postprocess,evaluate,criterion,trunk,decoder") == {
        "attention", "postprocess", "evaluate", "criterion", "trunk", "decoder"}
    assert _parse_groups("attention,postprocess,evaluate,criterion,trunk,decoder,transformer") == {
        "attention", "postprocess", "evaluate", "criterion", "trunk", "decoder", "transformer"}
    for bad in ("attention,dense", "attention,metrics", "criterion,loss", "trunk,voxel", "decoder,prune",
                "transformer,glue"):
        with pytest.raises(ValueError) as e:
            _parse_groups(bad)
        assert str(e.value) == (f"PASCO_B200_HOOKS={bad!r}: expected 0, 1 or a comma list of attention, postprocess, "
                                "evaluate, criterion, trunk, decoder, transformer")
    assert all(triggers for triggers, _ in _GROUPS.values())


def _start(code: str, value):
    env = {k: v for k, v in os.environ.items() if k != "PASCO_B200_HOOKS"}
    if value is not None:
        env["PASCO_B200_HOOKS"] = value
    python = [sys.executable] + (["-s"] if sys.flags.no_user_site else [])
    return subprocess.Popen(python + ["-c", PATHS + code], env=env, cwd=ROOT, text=True, stdout=subprocess.PIPE,
                            stderr=subprocess.STDOUT)


@pytest.mark.parametrize("value", [None, "1", "attention,trunk", "attention,bogus"])
def test_first_import_parses_the_switch(value):
    code = ("try:\n    import {}\nexcept ValueError as e:\n    print('ValueError', e)\nelse:\n    print('imported')\n")
    procs = {first: _start(code.format(first), value) for first in FIRST}
    outs = {first: p.communicate(timeout=300)[0] for first, p in procs.items()}
    for first, p in procs.items():
        assert p.returncode == 0, (first, outs[first])
        last = outs[first].strip().splitlines()[-1]
        if value == "attention,bogus":
            assert last.startswith("ValueError PASCO_B200_HOOKS='attention,bogus'"), (first, outs[first])
        else:
            assert last == "imported", (first, outs[first])


@pytest.mark.skipif(not os.path.isdir(os.path.join(REF, "pasco")), reason="oracle/_ref not staged")
def test_requested_groups_install_on_the_first_sparse_tensor():
    code = """
import torch
import MinkowskiEngine as ME
from pasco_b200 import hooks
import pasco.models.transformer.transformer_predictor_v2, pasco.models.augmenter, pasco.loss.criterion_sparse
from pasco.models.unet3d_sparse_v2 import CylinderFeat
import pasco.loss.losses
assert hooks._installed == set() and CylinderFeat.forward is not hooks._cylinder_forward
try:
    ME.SparseTensor(torch.zeros(1, 2), torch.zeros(1, 4, dtype=torch.int32))
except Exception:
    pass                        # no CUDA tensors here: the hooks install before the coordinates are read
assert hooks._installed == {"attention", "trunk", "criterion"}, hooks._installed
assert CylinderFeat.forward is hooks._cylinder_forward
print("installed")
"""
    p = _start(code, "attention,trunk,criterion")
    out = p.communicate(timeout=300)[0]
    assert p.returncode == 0 and out.strip().splitlines()[-1] == "installed", out
