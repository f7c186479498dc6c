"""CPU: the typed ragged entry points (r8bgpu_batch_process_ragged_fmt / _host_ragged_fmt) as the header declares them,
as the Python binding binds them, and as the r8b:: front-end calls them."""
import ctypes as C
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
NAMES = ("r8bgpu_batch_process_ragged_fmt", "r8bgpu_batch_process_host_ragged_fmt")


def _pkg():
    from __graft_entry__ import load_package
    return load_package()


def _declared(name):
    with open(os.path.join(ROOT, "include", "r8bgpu.h")) as f:
        text = f.read()
    m = re.search(r"R8BGPU_API\s+(\w+)\s+" + name + r"\s*\(([^;]*)\)\s*;", text)
    assert m, name + " is not declared"
    args = [" ".join(a.split()) for a in m.group(2).split(",")]
    return m.group(1), args


def _ctype(decl):
    if "*" in decl:
        return C.c_void_p
    return {"int": C.c_int, "size_t": C.c_size_t}[decl.rsplit(" ", 1)[0].replace("const ", "")]


@pytest.mark.parametrize("name", NAMES)
def test_header_and_binding_agree(name):
    ret, args = _declared(name)
    assert ret == "int"
    assert args[0] == "r8bgpu_batch* batch"
    assert [a.rsplit(" ", 1)[0] for a in args[1:]] == ["const r8bgpu_buffer*", "const int*", "const r8bgpu_buffer*", "int", "int*"]
    res, argtypes = _pkg()._SYMBOLS[name]
    assert res is C.c_int
    assert argtypes == [_ctype(a) for a in args]


def test_front_end_overloads_compile(tmp_path):
    gxx = shutil.which("g++")
    if gxx is None:
        pytest.skip("no g++")
    src = tmp_path / "use.cpp"
    src.write_text(
        '#include "r8b/CDSPResampler.h"\n'
        "int use(r8b::CDSPResamplerBatch& b, const r8bgpu_buffer& i, const int* lens, const r8bgpu_buffer& o, int* counts)\n"
        "{\n"
        "    return b.processRagged(i, lens, o, 16, counts) + b.processRaggedDevice(i, lens, o, 16, counts);\n"
        "}\n")
    r = subprocess.run([gxx, "-std=c++11", "-fsyntax-only", "-Wall", "-I", os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
