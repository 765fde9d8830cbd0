"""In-place kernels for wide ops (VERDICT r1 row 16 / #7): dense blocks on 5..10 qubits and diagonals on 5..10 qubits
against the CPU oracle (oracle/qip_oracle.c == qip-iterators/src/matrix_ops.rs:62-152)."""
import numpy as np
import pytest

from rustqip_b200.ops import make_control_op, make_matrix_op
from rustqip_b200.state import State

from test_gpu_parity import assert_close, oracle_apply, rand_state, rand_unitary

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("dtype", [np.complex128, np.complex64])
def test_wide_dense_and_diagonal_in_place(ctx, dtype):
    """Dense blocks on 5..8 qubits and diagonals on 5..9 qubits run IN PLACE (k_dense5 / k_dense_big / k_diag_wide),
    on every range of bit positions, with unordered indices and with controls: the reference applies any k through
    the same row loop (qip-iterators/src/iterators/qubit_iterators.rs:23-55, matrix_ops.rs:62-94)."""
    n = 13
    rng = np.random.default_rng(77)
    psi = rand_state(n, dtype, 15)
    cases = []
    for k in (5, 6):
        u = rand_unitary(k, rng)
        for lo in range(0, n - k + 1, 2):  # contiguous windows over the whole index
            qs = list(range(lo, lo + k))
            rng.shuffle(qs)
            cases.append(make_matrix_op(qs, u.reshape(-1)))
        for _ in range(3):  # scattered, unordered
            cases.append(make_matrix_op([int(q) for q in rng.choice(n, k, replace=False)], u.reshape(-1)))
    for k in (7, 8):
        cases.append(make_matrix_op([int(q) for q in rng.choice(n, k, replace=False)], rand_unitary(k, rng).reshape(-1)))
    q = [int(x) for x in rng.choice(n, 8, replace=False)]
    cases.append(make_control_op([q[0]], make_matrix_op(q[1:6], rand_unitary(5, rng).reshape(-1))))
    cases.append(make_control_op([q[0], q[7]], make_matrix_op(q[1:7], rand_unitary(6, rng).reshape(-1))))
    for k in (5, 7, 9):
        qs = [int(x) for x in rng.choice(n, k, replace=False)]
        cases.append(make_matrix_op(qs, np.diag(np.exp(1j * rng.standard_normal(1 << k))).reshape(-1)))
    cases.append(make_control_op([q[2]], make_matrix_op([x for x in range(n) if x != q[2]][:6],
                                                        np.diag(np.exp(1j * rng.standard_normal(64))).reshape(-1))))
    with State(n, dtype, ctx) as st:
        for op in cases:
            want = oracle_apply(n, op, psi)
            st.upload(psi)
            l0 = ctx.kernel_launches()
            st.apply_op(op)
            assert ctx.kernel_launches() - l0 == 1
            assert_close(st.download(), want, dtype)


def test_wide_dense_f64_smallest_states(ctx):
    """The f64 5/6-qubit blocks go to the tensor pipe (k_dense_dmma) from 16 groups per shard on; below that the FMA
    kernels take over.  Both sides of the switch against the oracle.  The QIPB200_DENSE_DMMA=0 override is read once
    per process; tests/test_gpu_full_size.py::test_dense_f64_fma_kernels_with_dmma_off runs it in a child process."""
    rng = np.random.default_rng(78)
    for n, k in [(9, 5), (8, 5), (7, 5), (10, 6), (9, 6), (11, 6), (12, 5)]:
        psi = rand_state(n, np.complex128, 16 + n)
        qs = [int(q) for q in rng.choice(n, k, replace=False)]
        op = make_matrix_op(qs, rand_unitary(k, rng).reshape(-1))
        want = oracle_apply(n, op, psi)
        with State(n, np.complex128, ctx) as st:
            st.upload(psi)
            st.apply_op(op)
            assert_close(st.download(), want, np.complex128)
