"""The convolution consumers keep one wgmma group in flight (DESIGN.md §3.1).  That holds only if ptxas keeps each slot's
MMA chain and its commit together: when the MMAs sit in a branch and the commit after it, ptxas ends the chain in the
branch and commits an empty dummy group (`HGMMA.64x8x16 ... gdesc[URZ]`), so `wgmma.wait_group 1` leaves only the dummy
outstanding and every slot is drained again.  This checks the SASS of the built library (no GPU needed)."""
import re
import subprocess

import pytest


@pytest.fixture(scope="module")
def sass():
    from pasco_b200 import build, _lib
    build.build()
    return subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True, check=True).stdout


def _functions(sass, name):
    out, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = m.group(1) if name in m.group(1) else None
            if cur:
                out[cur] = []
        elif cur:
            out[cur].append(line)
    return out


@pytest.mark.parametrize("kernel", ["k_conv_pl", "k_conv_tc"])
def test_conv_consumers_wait_for_all_but_the_last_real_mma_group(sass, kernel):
    funcs = _functions(sass, kernel)
    assert funcs, f"{kernel} not in the library"
    for name, lines in funcs.items():
        lagged, last_hgmma = 0, None
        for line in lines:
            if "HGMMA" in line:
                last_hgmma = line
            if re.search(r"WARPGROUP\.DEPBAR\.LE gsb0, 0x1\b", line):
                lagged += 1
                assert last_hgmma is not None and "gdesc[URZ]" not in last_hgmma, \
                    f"{name}: wait_group 1 follows an empty dummy MMA group: {last_hgmma.strip()}"
        assert lagged > 0, f"{name}: no wgmma.wait_group 1 (every slot drained)"
