"""Gate-schedule wire format and amplitude dump/load (SURVEY.md section 8f, row N3).

The reference's only export is OpenQASM 2.0 (qip/src/qasm.rs:112-184), which is lossy for this
path (MAT and GlobalPhase entries become comments).  These two little-endian binary formats
carry exactly what the C ABI consumes, so non-Rust callers and the bench harness can exchange
circuits and states:

schedule file ("QIPS", version 1)
    u32 magic 0x53504951 | u32 version | u32 prec (0 f32, 1 f64) | u32 n_qubits | u64 n_ops
    then n_ops records, each (recursive for Control):
      u8 kind (0 Matrix, 1 SparseMatrix, 2 Swap, 3 Control) | u32 n_indices | u32 n_control
      u64 indices[n_indices]
      Matrix:        u64 n_entries | complex<prec>[n_entries]   (row-major 4^k, ops.rs:13)
      SparseMatrix:  u64 n_rows | per row: u64 nnz | nnz x (u64 col, complex<prec> val)
      Swap:          -                                           (indices = a ++ b)
      Control:       one nested record (the inner op)

state file ("QIPA", version 1): one file per shard
    u32 magic 0x41504951 | u32 version | u32 prec | u32 n_qubits | u32 rank | u32 world
    u64 first_index | u64 n_amplitudes | complex<prec>[n_amplitudes]
"""
from __future__ import annotations

import struct
from typing import BinaryIO, List, Sequence, Tuple

import numpy as np

from ._abi import QIP_F32, QIP_F64, cdtype, prec_of
from .errors import CircuitError
from .ops import MatrixOp

MAGIC_SCHEDULE = 0x53504951
MAGIC_STATE = 0x41504951
_KIND = {"matrix": 0, "sparse": 1, "swap": 2, "control": 3}


def _w_op(f: BinaryIO, op: MatrixOp, dt) -> None:
    idx = op.indices()
    f.write(struct.pack("<BII", _KIND[op.kind], len(idx), op.n_control if op.kind == "control" else 0))
    f.write(np.asarray(idx, dtype="<u8").tobytes())
    if op.kind == "matrix":
        d = np.ascontiguousarray(np.asarray(op.data).reshape(-1).astype(dt))
        f.write(struct.pack("<Q", d.shape[0]))
        f.write(d.tobytes())
    elif op.kind == "sparse":
        f.write(struct.pack("<Q", len(op.rows)))
        for row in op.rows:
            f.write(struct.pack("<Q", len(row)))
            for c, v in row:
                f.write(struct.pack("<Q", c))
                f.write(np.asarray([v], dtype=dt).tobytes())
    elif op.kind == "control":
        _w_op(f, op.inner, dt)


def _r_exact(f: BinaryIO, n: int) -> bytes:
    b = f.read(n)
    if len(b) != n:
        raise CircuitError("schedule file truncated")
    return b


def _r_op(f: BinaryIO, dt) -> MatrixOp:
    kind, n_idx, n_ctrl = struct.unpack("<BII", _r_exact(f, 9))
    idx = [int(x) for x in np.frombuffer(_r_exact(f, 8 * n_idx), dtype="<u8")]
    size = np.dtype(dt).itemsize
    if kind == 0:
        (n_ent,) = struct.unpack("<Q", _r_exact(f, 8))
        data = np.frombuffer(_r_exact(f, size * n_ent), dtype=dt).copy()
        return MatrixOp.new_matrix(idx, data)
    if kind == 1:
        (n_rows,) = struct.unpack("<Q", _r_exact(f, 8))
        rows = []
        for _ in range(n_rows):
            (nnz,) = struct.unpack("<Q", _r_exact(f, 8))
            row = []
            for _ in range(nnz):
                (c,) = struct.unpack("<Q", _r_exact(f, 8))
                v = np.frombuffer(_r_exact(f, size), dtype=dt)[0]
                row.append((int(c), complex(v)))
            rows.append(row)
        return MatrixOp.new_sparse(idx, rows)
    if kind == 2:
        half = n_idx // 2
        return MatrixOp.new_swap(idx[:half], idx[half:])
    if kind == 3:
        inner = _r_op(f, dt)
        return MatrixOp("control", idx, n_control=n_ctrl, inner=inner)
    raise CircuitError("schedule file: unknown op kind %d" % kind)


def dump_schedule(path: str, n_qubits: int, ops: Sequence[MatrixOp], dtype=np.complex128) -> None:
    prec = prec_of(dtype)
    dt = cdtype(prec)
    with open(path, "wb") as f:
        f.write(struct.pack("<IIIIQ", MAGIC_SCHEDULE, 1, prec, n_qubits, len(ops)))
        for op in ops:
            _w_op(f, op, dt)


def load_schedule(path: str) -> Tuple[int, type, List[MatrixOp]]:
    with open(path, "rb") as f:
        magic, version, prec, n, n_ops = struct.unpack("<IIIIQ", _r_exact(f, 24))
        if magic != MAGIC_SCHEDULE or version != 1 or prec not in (QIP_F32, QIP_F64):
            raise CircuitError("not a QIPS version-1 schedule file")
        dt = cdtype(prec)
        return n, dt, [_r_op(f, dt) for _ in range(n_ops)]


def loads_schedule(data: bytes) -> Tuple[int, type, List[MatrixOp]]:
    """load_schedule of QIPS bytes held in memory."""
    import io

    f = io.BytesIO(data)
    magic, version, prec, n, n_ops = struct.unpack("<IIIIQ", _r_exact(f, 24))
    if magic != MAGIC_SCHEDULE or version != 1 or prec not in (QIP_F32, QIP_F64):
        raise CircuitError("not a QIPS version-1 schedule")
    dt = cdtype(prec)
    ops = [_r_op(f, dt) for _ in range(n_ops)]
    if f.read(1):
        raise CircuitError("schedule: trailing bytes after the last record")
    return n, dt, ops


class ParsedSchedule:
    """A QIPS buffer parsed by the C ABI (`qipb200_schedule_parse`, rustqip_b200/csrc/wire.cpp): the library owns
    the `qip_op` records; `State.apply_marshalled(sched.ops, sched.n_ops)` runs them without a Python op tree."""

    def __init__(self, data: bytes):
        import ctypes as C

        from . import _lib

        L = _lib.lib()
        self._L = L
        self._h = C.c_void_p()
        err = C.create_string_buffer(256)
        buf = (C.c_ubyte * len(data)).from_buffer_copy(data)
        st = L.qipb200_schedule_parse(buf, len(data), C.byref(self._h), err, len(err))
        if st != 0:
            self._h = None
            raise CircuitError(err.value.decode("utf-8", "replace") or "malformed QIPS schedule", status=st)
        n_ops, n, prec = C.c_size_t(), C.c_uint32(), C.c_int()
        self.ops = L.qipb200_schedule_ops(self._h, C.byref(n_ops), C.byref(n), C.byref(prec))
        self.n_ops, self.n_qubits, self.prec = n_ops.value, n.value, prec.value

    def serialise(self) -> bytes:
        import ctypes as C

        need = self._L.qipb200_schedule_serialise(self.prec, self.n_qubits, self.ops, self.n_ops, None, 0)
        out = (C.c_ubyte * need)()
        got = self._L.qipb200_schedule_serialise(self.prec, self.n_qubits, self.ops, self.n_ops, out, need)
        if got != need or need == 0:
            raise CircuitError("qipb200_schedule_serialise failed")
        return bytes(out)

    def close(self):
        if self._h:
            self._L.qipb200_schedule_free(self._h)
            self._h = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()


def serialise_ops(n_qubits: int, ops: Sequence[MatrixOp], dtype=np.complex128) -> bytes:
    """QIPS bytes written by the C ABI from marshalled `qip_op` records (the writer a Rust/C caller uses)."""
    import ctypes as C

    from . import _lib
    from ._abi import marshal_ops

    prec = prec_of(dtype)
    arr, keep = marshal_ops(ops, prec)
    L = _lib.lib()
    need = L.qipb200_schedule_serialise(prec, n_qubits, arr, len(ops), None, 0)
    if need == 0:
        raise CircuitError("qipb200_schedule_serialise failed")
    out = (C.c_ubyte * need)()
    if L.qipb200_schedule_serialise(prec, n_qubits, arr, len(ops), out, need) != need:
        raise CircuitError("qipb200_schedule_serialise failed")
    return bytes(out)


def dump_state(path: str, state) -> None:
    """Write this rank's shard of a device-resident `State` (canonical layout)."""
    amps = state.download()
    with open(path, "wb") as f:
        f.write(struct.pack("<IIIIIIQQ", MAGIC_STATE, 1, state.prec, state.n, state.rank, state.world_size,
                            state.rank * state.local_len, amps.shape[0]))
        f.write(np.ascontiguousarray(amps).tobytes())


def load_state(path: str, state) -> None:
    """Upload a shard written by dump_state into a `State` of the same shape."""
    with open(path, "rb") as f:
        magic, version, prec, n, rank, world, first, count = struct.unpack("<IIIIIIQQ", _r_exact(f, 40))
        if magic != MAGIC_STATE or version != 1:
            raise CircuitError("not a QIPA version-1 state file")
        if (prec, n, rank, world) != (state.prec, state.n, state.rank, state.world_size) or count != state.local_len:
            raise CircuitError("state file does not match the target state (prec/n/rank/world/length)")
        amps = np.frombuffer(_r_exact(f, count * np.dtype(state.dtype).itemsize), dtype=state.dtype)
    state.upload(amps)
