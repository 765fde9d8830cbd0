"""qipb200_state_sample without a GPU: argument checks at the C boundary and the C++ mirror's wrapper."""
import ctypes as C
import os
import subprocess

from rustqip_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
QIPB200_ERR_INVALID_ARG = 1


def test_sample_rejects_null_state():
    L = _lib.lib()
    out = (C.c_uint64 * 4)()
    draws = (C.c_double * 4)(0.1, 0.2, 0.3, 0.4)
    idx = (C.c_uint64 * 1)(0)
    assert L.qipb200_state_sample(None, idx, 1, draws, 4, out) == QIPB200_ERR_INVALID_ARG
    assert b"sample" in L.qipb200_last_error(None)
    assert L.qipb200_state_sample(None, None, 0, None, 0, None) == QIPB200_ERR_INVALID_ARG


def test_cpp_mirror_sample_compiles(tmp_path):
    src = tmp_path / "use_sample.cpp"
    src.write_text('#include "qipb200.hpp"\n'
                   "std::vector<uint64_t> shots(qip::B200State<double> &st) {\n"
                   "  return st.sample({0, 2}, {0.25, 0.5, 0.75});\n"
                   "}\n")
    p = subprocess.run(["/usr/bin/g++", "-std=c++17", "-fsyntax-only", "-I" + os.path.join(ROOT, "include"), str(src)],
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr
