"""The f64 tile geometry of states on generated kernels (L = 4: 256-byte contiguous runs, 8 free tile bits), checked
without a GPU: the planner's choice and the host-compiled generated kernels at T = 12 / L = 4 against the oracle."""
import ctypes as C
import os
import tempfile

import numpy as np
import pytest

from oracle import qip_oracle as qo
from rustqip_b200 import circuits, gates
from rustqip_b200._abi import QipOp, marshal_ops, prec_of
from test_jit_cpu import emul, rand_state  # noqa: F401  (emul: the host-compiled generator fixture)

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.mark.parametrize("seed", [0x5EED0002, 0x5EED0003])
def test_generated_kernels_at_l4(emul, seed):  # noqa: F811
    n = 16
    ops = circuits.random_circuit(n, 10, seed, "H,T,CNOT") + circuits.qft(n)[:40]
    rng = np.random.default_rng(seed)
    for _ in range(20):
        a, b, c = [int(x) for x in rng.choice(n, 3, replace=False)]
        ops += [gates.toffoli(a, b, c), gates.cz(a, b), gates.rz(c, 0.3)]
    psi = rand_state(n, 5, np.complex128)
    want = qo.run_pipeline(n, ops, state=psi, dtype=np.complex128)
    arr, keep = marshal_ops(ops, prec_of(np.complex128))
    st = np.ascontiguousarray(psi)
    stats = np.zeros(8, dtype=np.uint64)
    err = C.create_string_buffer(512)
    with tempfile.TemporaryDirectory() as d:
        rc = emul.emul_schedule_jit(prec_of(np.complex128), n, arr, len(ops), st.ctypes.data, 12, 4, d.encode(),
                                    stats.ctypes.data, err, 512)
    assert rc == 0, err.value
    assert stats[0] >= 2 and stats[1] == 0
    assert np.max(np.abs(st - want)) <= 1e-11 * np.max(np.abs(want))


def test_headline_circuit_sweeps(monkeypatch):
    """N = 30 f64, depth-40 {H, T, CNOT}: 21 passes at the default L = 4 (25 at L = 5), every one covered by the
    generator; with the generated kernels off the interpreter keeps L = 5."""
    for var in ("QIPB200_JIT", "QIPB200_TILE_T", "QIPB200_TILE_L", "QIPB200_JIT_GROUP_BITS"):
        monkeypatch.delenv(var, raising=False)
    L = C.CDLL(os.path.join(HERE, "native", "_build", "libplan_emul.so"))
    L.emul_plan_stats.restype = C.c_int
    L.emul_plan_stats.argtypes = [C.c_int, C.c_uint32, C.POINTER(QipOp), C.c_size_t, C.c_uint32, C.c_uint32, C.c_int,
                                  C.c_uint32, C.c_void_p]
    L.emul_jit_plan_stats.restype = C.c_int
    L.emul_jit_plan_stats.argtypes = [C.c_int, C.c_uint32, C.POINTER(QipOp), C.c_size_t, C.c_int, C.c_void_p]
    ops = circuits.random_circuit(30, 40, 0x5EED0002)
    arr, keep = marshal_ops(ops, prec_of(np.complex128))

    def sweeps():
        st = np.zeros(64, dtype=np.uint64)
        assert L.emul_plan_stats(prec_of(np.complex128), 30, arr, len(ops), 0, 0, 1, 0, st.ctypes.data) == 0
        assert st[1] == 0
        return st

    assert sweeps()[0] == 21
    js = np.zeros(8, dtype=np.uint64)
    assert L.emul_jit_plan_stats(prec_of(np.complex128), 30, arr, len(ops), 0, js.ctypes.data) == 0
    assert js[0] == 21 and js[1] == 0
    monkeypatch.setenv("QIPB200_TILE_L", "5")
    assert sweeps()[0] == 25
    monkeypatch.delenv("QIPB200_TILE_L")
    monkeypatch.setenv("QIPB200_JIT", "off")
    assert sweeps()[0] > 21
