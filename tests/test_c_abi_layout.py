"""The ctypes mirrors of the C ABI's structs (p2pvg_b200/_lib.py) against include/p2pvg_b200.h, as the host C++ compiler lays
them out.  A mismatch would only show up on the GPU, as pointers read from the wrong offsets."""
import ctypes
import os
import subprocess

import pytest

from p2pvg_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.parametrize("c_name,py_struct", [("p2pvg_conv_fusion_t", _lib.ConvFusion),
                                              ("p2pvg_lstm_step_module", _lib.LstmStepModule)])
def test_ctypes_struct_matches_the_header(tmp_path, c_name, py_struct):
    fields = [f[0] for f in py_struct._fields_]
    src = tmp_path / "layout.cpp"
    src.write_text('#include <cstddef>\n#include <cstdio>\n#include "p2pvg_b200.h"\nint main() {\n'
                   f'  std::printf("sizeof %zu\\n", sizeof({c_name}));\n'
                   + "".join(f'  std::printf("{f} %zu\\n", offsetof({c_name}, {f}));\n' for f in fields) + "}\n")
    exe = tmp_path / "layout"
    subprocess.run(["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout
    got = dict((k, int(v)) for k, v in (line.split() for line in out.splitlines()))
    want = {"sizeof": ctypes.sizeof(py_struct), **{f: getattr(py_struct, f).offset for f in fields}}
    assert got == want
