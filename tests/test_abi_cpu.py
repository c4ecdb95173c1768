"""The C-ABI library loads without a GPU and exports every symbol include/svgb200.h declares; argument
errors come back as rc < 0 with a message (no compute calls here)."""
import ctypes as C
import re
from pathlib import Path

import pytest

ROOT = Path(__file__).resolve().parent.parent


@pytest.fixture(scope="module")
def lib():
    import importlib.util

    spec = importlib.util.spec_from_file_location("svgb200_build", ROOT / "sparse-videogen_b200" / "build.py")
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    mod.build_lib()
    from svgb200 import _lib

    return _lib.lib()


def test_exports_every_declared_symbol(lib):
    header = (ROOT / "include" / "svgb200.h").read_text()
    names = sorted(set(re.findall(r"\b(svgb_[a-z0-9_]+)\s*\(", header)))
    assert len(names) >= 23
    for n in names:
        assert hasattr(lib, n), f"{n} declared in svgb200.h but not exported"
    assert lib.svgb_version() >= 100


def test_prototypes_cover_the_header(lib):
    from svgb200 import _lib

    header = (ROOT / "include" / "svgb200.h").read_text()
    names = set(re.findall(r"\b(svgb_[a-z0-9_]+)\s*\(", header)) - {"svgb_last_error"}
    assert names == set(_lib._PROTOS), names ^ set(_lib._PROTOS)


def test_argument_errors_are_reported(lib):
    n = C.c_size_t()
    assert lib.svgb_attn_plan_varblock_bytes(0, 10, 1, 1, C.byref(n)) < 0
    assert b"bad arguments" in lib.svgb_last_error()
    assert lib.svgb_attn_plan_varblock_bytes(24, 119056, 402, 1002, C.byref(n)) == 0 and n.value > 0
    assert lib.svgb_kmeans_bytes(2, 100, 5000, 128, C.byref(n)) < 0
    assert lib.svgb_sample_mse_bytes(2, 1000, 96, 64, C.byref(n)) < 0


def test_plan_struct_mirrors_header():
    """_lib.Plan declares the fields of `struct svgb_plan` in include/svgb200.h, in order and with their types."""
    from svgb200._lib import Plan

    header = (ROOT / "include" / "svgb200.h").read_text()
    body = re.search(r"typedef struct svgb_plan \{(.*?)\} svgb_plan;", header, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    ctype = {"int32_t": C.c_int32, "int64_t": C.c_int64}
    fields = [(name.strip(), ctype[t]) for t, names in re.findall(r"(int32_t|int64_t)\s+([^;]+);", body)
              for name in names.split(",")]
    assert fields == list(Plan._fields_)
    assert C.sizeof(Plan) == 9 * 4 + 4 + 4 * 8  # 4 bytes of padding align the first int64
    assert Plan.counts_off.offset == 40


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from svgb200 import _lib

    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "_LIB_PATH", tmp_path / "nope.so")
    with pytest.raises(_lib.SvgbError):
        _lib.lib()


def test_cpu_tensors_are_rejected():
    import torch

    from svgb200 import core

    with pytest.raises(core.SvgbError):
        core.permute_gather(torch.zeros(1, 4, 8, dtype=torch.bfloat16), torch.zeros(1, 4, dtype=torch.int32))
