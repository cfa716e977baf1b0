"""CPU-side checks of the drop-in boundary: the C-ABI library builds, loads and exports every
symbol include/pasco_sm100.h declares; the product never routes through the oracle; ops fail
loudly without a GPU."""
import os
import re
import subprocess
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from pasco_b200 import build, _lib
    build.build()
    return _lib.load()


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "pasco_sm100.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(pasco_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_are_exported_and_typed(lib):
    from pasco_b200 import _lib
    names = _declared_symbols()
    assert len(names) >= 25
    for n in names:
        assert hasattr(lib, n), f"{n} declared in include/pasco_sm100.h but not exported"
        assert n in _lib.PROTOTYPES, f"{n} has no ctypes prototype"
    assert sorted(_lib.PROTOTYPES) == names, "ctypes prototypes and header disagree"


def test_header_declarations_match_ctypes_prototypes():
    """Every pasco_* declaration's return and argument kinds equal _lib.PROTOTYPES: pointers, arrays and the stream →
    c_void_p, `const char*` → c_char_p, the scalar types → their ctypes types."""
    from pasco_b200 import _lib
    C = _lib.C
    scalar = {"int": C.c_int, "int32_t": C.c_int32, "int64_t": C.c_int64, "uint64_t": C.c_uint64, "float": C.c_float,
              "double": C.c_double, "pasco_stream_t": C.c_void_p}

    def kind(text, ret=False):
        """ctypes type of a return type, or of one parameter (type and name)."""
        t = text.replace("const", " ")
        if not ret:                                  # drop the name; an array parameter is a pointer
            t = re.sub(r"\w+\s*(\[\d*\])?\s*$", lambda m: "" if m.group(1) is None else "*", t)
        words = t.replace("*", " * ").split()
        if "*" in words:
            return C.c_char_p if ret and words[0] == "char" else C.c_void_p
        return scalar[words[0]]

    src = re.sub(r"/\*.*?\*/|//[^\n]*", "", open(os.path.join(ROOT, "include", "pasco_sm100.h")).read(), flags=re.S)
    decls = re.findall(r"([\w\s\*]+?)\b(pasco_[a-z0-9_]+)\s*\(([^;{)]*)\)\s*;", src)
    assert sorted(name for _, name, _ in decls) == _declared_symbols()
    for ret, name, args in decls:
        want = (kind(ret, ret=True), [kind(a) for a in args.split(",") if a.strip() not in ("", "void")])
        assert want == _lib.PROTOTYPES[name], (name, want, _lib.PROTOTYPES[name])


def test_abi_version_3_and_error_string(lib):
    assert lib.pasco_abi_version() == 3
    assert isinstance(lib.pasco_last_error(), bytes)
    assert lib.pasco_conv_packed_bytes(27, 64, 64) == 27 * 64 * 64 * 4


def test_library_is_sm90a_with_wgmma_and_bulk_copy(lib):
    from pasco_b200 import _lib
    sass = subprocess.run(["cuobjdump", "-sass", _lib.LIB_PATH], capture_output=True, text=True).stdout
    assert "arch = sm_90a" in sass
    assert "HGMMA" in sass, "no wgmma in the SASS"
    assert "SYNCS" in sass, "no mbarrier in the SASS"
    assert "UBLKCP" in sass, "no bulk async copy in the SASS"


def test_product_never_imports_the_oracle():
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pasco_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "me_oracle" not in txt and "oracle." not in txt.replace("the oracle.", ""), f
    txt = open(os.path.join(ROOT, "compat", "MinkowskiEngine", "__init__.py")).read()
    assert "me_oracle" not in txt


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_ops_fail_loudly_without_a_gpu(lib):
    from pasco_b200 import me
    with pytest.raises((AssertionError, RuntimeError)):
        me.SparseTensor(torch.zeros(2, 4), torch.zeros(2, 4, dtype=torch.int32))
    from pasco_b200._lib import call, PascoError
    with pytest.raises(PascoError):
        call("pasco_hash_remap", None, 0, None)
