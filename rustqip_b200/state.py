"""Device context and device-resident state handles (thin RAII over the C ABI).

``State`` plays the role of the two ``Vec<Complex<P>>`` owned by
``LocalBuilder::calculate_state_with_init`` (qip/src/builder.rs:406-407): the
amplitudes stay in HBM between gates; only explicit download copies them out.
"""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional, Sequence

import numpy as np

from . import _lib
from ._abi import QIP_F32, QIP_F64, cdtype, marshal_op, marshal_ops, prec_of
from .errors import B200Unavailable, CircuitError
from .ops import MatrixOp


class Context:
    """One CUDA device + stream (qipb200_ctx).  One process per GPU."""

    def __init__(self, device=0):
        """device: one CUDA device id, or a list of ids (a power-of-two count): ONE context over several devices
        of this process (qipb200_init_multi) whose states are sharded over them inside the library."""
        self._h = C.c_void_p()
        L = _lib.lib()
        if isinstance(device, (list, tuple)):
            ids = (C.c_int * len(device))(*[int(d) for d in device])
            st = L.qipb200_init_multi(C.byref(self._h), len(device), ids)
            self.device = int(device[0])
            self.devices = [int(d) for d in device]
        else:
            st = L.qipb200_init(C.byref(self._h), int(device))
            self.device = int(device)
            self.devices = [int(device)]
        if st != 0:
            msg = L.qipb200_last_error(None).decode("utf-8", "replace")
            raise B200Unavailable(msg)

    @property
    def handle(self):
        return self._h

    def stream_handle(self) -> int:
        """Raw cudaStream_t of this context (for CUDA-event timing by the caller)."""
        sp = C.c_void_p()
        _lib.check(_lib.lib().qipb200_stream_handle(self._h, C.byref(sp)), self._h)
        return int(sp.value or 0)

    def launch_stats(self):
        """dict(all, tile_passes, exchanges, fused_gates) -- cumulative counters of this context."""
        out = (C.c_uint64 * 4)()
        _lib.check(_lib.lib().qipb200_launch_stats(self._h, out), self._h)
        return {"all": int(out[0]), "tile_passes": int(out[1]), "exchanges": int(out[2]), "fused_gates": int(out[3])}

    def jit_stats(self, wait: bool = False):
        """Generated-kernel statistics; wait=True blocks until the background NVRTC compilations are done."""
        out = (C.c_double * 4)()
        note = C.create_string_buffer(512)
        _lib.check(_lib.lib().qipb200_jit_stats(self._h, 1 if wait else 0, out, note, 512), self._h)
        return {"jit_passes": int(out[0]), "tile_passes": int(out[1]), "programs_compiled": int(out[2]),
                "compile_ms_total": out[3], "note": note.value.decode("utf-8", "replace")}

    def profile(self, on: bool):
        """Bracket every fused tile pass / NVLink exchange with CUDA events on the context's stream."""
        _lib.check(_lib.lib().qipb200_profile_enable(self._h, 1 if on else 0), self._h)

    def profile_read(self):
        """dict(tile_ms, tile_passes, exchange_ms, exchanges) since the previous read (synchronises the stream)."""
        out = (C.c_double * 4)()
        _lib.check(_lib.lib().qipb200_profile_read(self._h, out), self._h)
        return {"tile_ms": out[0], "tile_passes": int(out[1]), "exchange_ms": out[2], "exchanges": int(out[3])}

    def kernel_launches(self) -> int:
        return int(_lib.lib().qipb200_kernel_launches(self._h))

    KERNELS = ("k_dense", "k_diag", "k_diag_wide", "k_exchange", "k_dense5", "k_dense_dmma", "k_dense_big", "k_gather")

    def kernel_counts(self):
        """dict kernel name -> per-gate launches of that kernel so far (apply_op and unfused schedules)."""
        out = (C.c_uint64 * len(self.KERNELS))()
        _lib.check(_lib.lib().qipb200_kernel_counts(self._h, out, len(self.KERNELS)), self._h)
        return {k: int(v) for k, v in zip(self.KERNELS, out)}

    def release_pool(self):
        """Return the buffer kept from the last freed state to the device (the next state allocates afresh)."""
        _lib.check(_lib.lib().qipb200_release_pool(self._h), self._h)

    def close(self):
        if self._h:
            _lib.lib().qipb200_shutdown(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def __del__(self):  # pragma: no cover
        try:
            self.close()
        except Exception:
            pass


_default_ctx: Optional[Context] = None


def default_context() -> Context:
    global _default_ctx
    if _default_ctx is None:
        _default_ctx = Context(0)
    return _default_ctx


def _ptr(a: np.ndarray):
    return a.ctypes.data


class State:
    """Device-resident 2^n amplitudes (or one rank's shard of them)."""

    def __init__(self, n: int, dtype=np.complex128, ctx: Optional[Context] = None, rank: int = 0,
                 world_size: int = 1):
        self.ctx = ctx or default_context()
        self.n = int(n)
        self.prec = prec_of(dtype)
        self.dtype = cdtype(self.prec)
        self.rank, self.world_size = int(rank), int(world_size)
        self._h = C.c_void_p()
        L = _lib.lib()
        if world_size == 1:
            st = L.qipb200_state_new(self.ctx.handle, self.prec, self.n, C.byref(self._h))
        else:
            st = L.qipb200_state_new_sharded(self.ctx.handle, self.prec, self.n, self.rank,
                                             self.world_size, C.byref(self._h))
        _lib.check(st, self.ctx.handle)
        g = (self.world_size - 1).bit_length()
        self.local_len = 1 << (self.n - g)

    # -- lifecycle ------------------------------------------------------------
    def free(self):
        if self._h:
            _lib.lib().qipb200_state_free(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.free()

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass

    def _chk(self, st):
        _lib.check(st, self.ctx.handle)

    # -- builder.rs:409-421 ---------------------------------------------------
    def set_basis(self, index: int):
        self._chk(_lib.lib().qipb200_state_set_basis(self._h, int(index)))

    def upload(self, host: np.ndarray, offset: int = 0):
        host = np.ascontiguousarray(host, dtype=self.dtype)
        self._chk(_lib.lib().qipb200_state_upload(self._h, _ptr(host), int(offset), host.shape[0]))

    def download(self, out: Optional[np.ndarray] = None, offset: int = 0, length: Optional[int] = None):
        if length is None:
            length = (out.shape[0] if out is not None else self.local_len - offset)
        if out is None:
            out = np.empty(length, dtype=self.dtype)
        assert out.dtype == self.dtype and out.flags.c_contiguous
        self._chk(_lib.lib().qipb200_state_download(self._h, _ptr(out), int(offset), int(length)))
        return out

    def download_ptr(self, host_ptr: int, length: int, offset: int = 0):
        """Download into raw host memory (e.g. a pinned torch tensor's data_ptr())."""
        self._chk(_lib.lib().qipb200_state_download(self._h, C.c_void_p(host_ptr), int(offset), int(length)))

    # -- builder.rs:499,514 ---------------------------------------------------
    def apply_op(self, op: MatrixOp):
        cop, keep = marshal_op(op, self.prec)
        self._chk(_lib.lib().qipb200_state_apply_op(self._h, C.byref(cop)))

    def apply_schedule(self, ops: Sequence[MatrixOp], fusion: bool = True):
        arr, keep = marshal_ops(ops, self.prec)
        self.apply_marshalled(arr, len(ops), fusion)

    def apply_marshalled(self, arr, n_ops: int, fusion: bool = True):
        flags = _lib.SCHED_DEFAULT if fusion else _lib.SCHED_NO_FUSION
        self._chk(_lib.lib().qipb200_state_apply_schedule(self._h, arr, n_ops, flags))

    def norm2(self) -> float:
        v = C.c_double()
        self._chk(_lib.lib().qipb200_state_norm2(self._h, C.byref(v)))
        return v.value

    def sync(self):
        self._chk(_lib.lib().qipb200_state_sync(self._h))

    def max_abs_diff(self, other: "State") -> float:
        """max over amplitudes of max(|d re|, |d im|) against another state of the same shape (on the device)."""
        v = C.c_double()
        self._chk(_lib.lib().qipb200_state_max_abs_diff(self._h, other._h, C.byref(v)))
        return v.value

    # -- N3: QIPA state files through the C ABI (checkpoint / resume) ----------------
    def save(self, path: str):
        self._chk(_lib.lib().qipb200_state_save(self._h, str(path).encode()))

    def load(self, path: str):
        self._chk(_lib.lib().qipb200_state_load(self._h, str(path).encode()))

    # -- measurement_ops.rs ---------------------------------------------------
    def measure_probs(self, indices: Sequence[int]) -> np.ndarray:
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        out = np.zeros(1 << len(idx), dtype=np.float64)
        self._chk(_lib.lib().qipb200_state_measure_probs(self._h, _ptr(idx), len(idx), _ptr(out)))
        return out

    def measure_prob(self, measured: int, indices: Sequence[int]) -> float:
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        v = C.c_double()
        self._chk(_lib.lib().qipb200_state_measure_prob(self._h, int(measured), _ptr(idx), len(idx), C.byref(v)))
        return v.value

    def soft_measure(self, indices: Sequence[int], r: float) -> int:
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        m = C.c_uint64()
        self._chk(_lib.lib().qipb200_state_soft_measure(self._h, _ptr(idx), len(idx), float(r), C.byref(m)))
        return int(m.value)

    def sample(self, indices: Sequence[int], draws=None, shots: Optional[int] = None, rng=None) -> np.ndarray:
        """Many soft_measure draws on the uncollapsed state: out[k] == soft_measure(indices, draws[k]).

        Without ``draws``, ``shots`` uniforms in [0, 1) are drawn from ``rng`` (a numpy Generator; a fresh
        ``np.random.default_rng()`` when None).  Reads the state at most twice for any number of draws."""
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        if draws is None:
            if shots is None:
                raise ValueError("sample: give draws or shots")
            draws = (rng if rng is not None else np.random.default_rng()).random(int(shots))
        r = np.ascontiguousarray(np.asarray(draws, dtype=np.float64).reshape(-1))
        out = np.zeros(r.shape[0], dtype=np.uint64)
        self._chk(_lib.lib().qipb200_state_sample(self._h, _ptr(idx), len(idx), _ptr(r), r.shape[0], _ptr(out)))
        return out

    def collapse(self, indices: Sequence[int], measured: int, prob: float):
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        self._chk(_lib.lib().qipb200_state_collapse(self._h, _ptr(idx), len(idx), int(measured), float(prob)))

    def measure(self, indices: Sequence[int], r: Optional[float] = None, measured: Optional[int] = None,
                prob: Optional[float] = None, rng=None):
        """measure (measurement_ops.rs:190-214): draw an outcome, take its probability, collapse; returns (m, p).

        ``measured`` forces the outcome and ``prob`` (with ``measured`` only) its probability, as the reference's
        MeasuredCondition does.  Otherwise the outcome is drawn with ``r`` in [0, 1), or with ``rng.random()`` (a
        fresh ``np.random.default_rng()`` when None).  On an unsharded state the collapse costs no sweep of its own
        when the next call is a fused apply_schedule."""
        idx = np.ascontiguousarray(np.asarray(list(indices), dtype=np.uint64))
        flags = 0
        m, p = C.c_uint64(0), C.c_double(0.0)
        if measured is not None:
            flags |= _lib.MEASURE_FORCED
            m.value = int(measured)
            if prob is not None:
                flags |= _lib.MEASURE_FORCED_PROB
                p.value = float(prob)
        elif prob is not None:
            raise ValueError("measure: prob is only taken with measured")
        elif r is None:
            r = (rng if rng is not None else np.random.default_rng()).random()
        self._chk(_lib.lib().qipb200_state_measure(self._h, _ptr(idx), len(idx), float(r or 0.0), flags, C.byref(m),
                                                   C.byref(p)))
        return int(m.value), float(p.value)

    def expect_paulis(self, terms) -> np.ndarray:
        """<psi|P_t|psi> for each Pauli string P_t on the state as it is (not renormalised), computed on the device.

        A term is a sequence of (letter, qubit) pairs with letters "X", "Y", "Z", e.g. ``[("Z", 0), ("Z", 1)]``; an
        empty term is the identity.  A read sweep of the state carries up to 16384 terms: terms with equal X/Y masks
        share one, Z-only terms ride along (``expect_plan`` gives the count).  For H = sum_t c_t P_t take ``np.dot(c, st.expect_paulis(P))``."""
        qs, ls, lens = _marshal_paulis(terms)
        out = np.zeros(max(1, lens.shape[0]), dtype=np.float64)
        self._chk(_lib.lib().qipb200_state_expect_paulis(self._h, _ptr(qs), ls, _ptr(lens), lens.shape[0], _ptr(out)))
        return out[: lens.shape[0]]

    def transition_paulis(self, ket: "State", terms) -> np.ndarray:
        """<self|P_t|ket> (complex128) for each Pauli string P_t, on the two states as they are (not renormalised),
        computed on the device; this state is the bra.

        Terms are encoded as for ``expect_paulis``; an empty term gives the overlap <self|ket>.  ``ket`` must be a
        state of the same context, precision and size (it may be this state).  Pending collapses are applied first;
        states with the same qubit layout are read where they are, otherwise each permuted one is restored first.  A
        read sweep of both states carries up to 8192 terms (``transition_plan`` gives the counts); deterministic;
        synchronises.  For <phi|H|psi> with H = sum_t c_t P_t take ``np.dot(c, phi.transition_paulis(psi, P))``."""
        qs, ls, lens = _marshal_paulis(terms)
        out = np.zeros(max(1, 2 * lens.shape[0]), dtype=np.float64)
        self._chk(_lib.lib().qipb200_state_transition_paulis(self._h, ket._h, _ptr(qs), ls, _ptr(lens), lens.shape[0],
                                                             _ptr(out)))
        return out[: 2 * lens.shape[0]].view(np.complex128)

    def overlap(self, ket: "State") -> complex:
        """<self|ket> on the device (``transition_paulis`` of the empty term); the fidelity of two normalised states
        is ``abs(a.overlap(b)) ** 2``."""
        return complex(self.transition_paulis(ket, [[]])[0])

    def apply_pauli_rotations(self, terms, angles):
        """Apply exp(-i angles[t]/2 P_t) for each Pauli string P_t, term 0 first, on the device.

        Terms are encoded as for ``expect_paulis``; a single ``[("Z", q)]`` term is ``gates.rz(q, angle)`` and a
        single ``[("X", q)]`` term is Rx(angle).  A read-write sweep of the state carries a run of consecutive terms
        whose X/Y letters fit one tile (``pauli_rotation_plan`` gives the count).  Stream-ordered like
        ``apply_schedule``; the result is the same bits however the terms are split over calls."""
        args = _pauli_args("apply_pauli_rotations", terms, angles, "angles")
        self._chk(_lib.lib().qipb200_state_apply_pauli_rotations(self._h, *args))

    def apply_channels(self, channels, qubits: Sequence[int], rng=None, draws=None):
        """One quantum-trajectory step of single-qubit channels on distinct qubits, computed on the device: each
        channel applies one of its Kraus operators, drawn with its Born probability, and the state is renormalised.
        Returns (chosen, prob): chosen[c] indexes the operator of channel c, prob is the probability of that tuple.

        ``channels`` is a ``channels.Channel`` for every qubit or one per qubit.  ``draws`` are 1 + len(qubits)
        uniforms in [0, 1) (draws[0] samples the state-dependent qubits as ``sample`` does, draws[1 + c] picks channel
        c's operator); without them they are drawn from ``rng`` (a fresh ``np.random.default_rng()`` when None).  At
        most three read sweeps and one read-write sweep whatever the number of channels (``channels_plan``);
        synchronises.  Averaging over trajectories reproduces the channels' density matrix."""
        from . import channels as _ch
        qa = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        chans = [channels] * qa.shape[0] if isinstance(channels, _ch.Channel) else list(channels)
        if len(chans) != qa.shape[0]:
            raise ValueError("apply_channels: %d channels but %d qubits" % (len(chans), qa.shape[0]))
        _single_qubit("apply_channels", chans, "apply_multiqubit_channels")
        _, n_kraus, kraus = _ch.marshal(chans)
        if draws is None:
            draws = (rng if rng is not None else np.random.default_rng()).random(1 + qa.shape[0])
        r = np.ascontiguousarray(np.asarray(draws, dtype=np.float64).reshape(-1))
        if r.shape[0] != 1 + qa.shape[0]:
            raise ValueError("apply_channels: %d channels need %d draws, got %d" % (qa.shape[0], 1 + qa.shape[0],
                                                                                   r.shape[0]))
        chosen = np.zeros(max(1, qa.shape[0]), dtype=np.uint32)
        prob = C.c_double()
        n = qa.shape[0]
        self._chk(_lib.lib().qipb200_state_apply_channels(self._h, n, _ptr(qa) if n else None,
                                                          _ptr(n_kraus) if n else None, _ptr(kraus) if n else None,
                                                          _ptr(r), _ptr(chosen), C.byref(prob)))
        return chosen[:n], float(prob.value)

    def apply_multiqubit_channels(self, channels, qubit_groups, rng=None, draws=None):
        """One quantum-trajectory step of channels on one to four qubits each, no qubit twice in the layer, computed
        on the device as ``apply_channels`` does.  Returns (chosen, prob).

        ``qubit_groups[c]`` lists the qubits of channel c, its first qubit the most significant bit of the channel's
        matrices; ``channels`` is one ``channels.Channel`` for every group or one per group, each on as many qubits as
        its group.  ``draws`` are 1 + len(qubit_groups) uniforms in [0, 1) (draws[0] samples the state-dependent
        channels' qubits, draws[1 + c] picks channel c's operator); without them they are drawn from ``rng``.  At most
        three read sweeps and one read-write sweep whatever the layer (``multiqubit_channels_plan``); synchronises.
        A layer of single-qubit channels gives the same bits as ``apply_channels``."""
        chans, qa = _channel_groups("apply_multiqubit_channels", channels, qubit_groups)
        arity, n_kraus, kraus = _ch_marshal(chans)
        nc = len(chans)
        if draws is None:
            draws = (rng if rng is not None else np.random.default_rng()).random(1 + nc)
        r = np.ascontiguousarray(np.asarray(draws, dtype=np.float64).reshape(-1))
        if r.shape[0] != 1 + nc:
            raise ValueError("apply_multiqubit_channels: %d channels need %d draws, got %d" % (nc, 1 + nc, r.shape[0]))
        chosen = np.zeros(max(1, nc), dtype=np.uint32)
        prob = C.c_double()
        self._chk(_lib.lib().qipb200_state_apply_multiqubit_channels(
            self._h, nc, _ptr(arity) if nc else None, _ptr(qa) if nc else None, _ptr(n_kraus) if nc else None,
            _ptr(kraus) if nc else None, _ptr(r), _ptr(chosen), C.byref(prob)))
        return chosen[:nc], float(prob.value)

    def apply_kraus_channels(self, channels, qubit_groups, rng=None, draws=None):
        """One quantum-trajectory step of channels with any complete Kraus sets on one to four qubits each, no qubit
        twice in the layer, computed on the device.  Returns (chosen, cond, prob): chosen[c] indexes the operator of
        channel c, cond[c] is the probability of that choice given the earlier ones, prob their product.

        ``qubit_groups[c]`` lists the qubits of channel c, its first qubit the most significant bit of the channel's
        matrices; ``channels`` is one ``channels.KrausChannel`` (or ``Channel``) for every group or one per group.
        ``draws`` are len(qubit_groups) uniforms in [0, 1), one per channel; without them they are drawn from ``rng``.
        State-independent channels (mixed-unitary ones) are drawn without reading the state and applied through
        ``apply_schedule``; the others cost one read sweep plus one read-write sweep per group of at most four qubits
        (``kraus_channels_plan``).  Monomial layers are cheaper through ``apply_multiqubit_channels``.  Synchronises."""
        chans, qa = _kraus_groups("apply_kraus_channels", channels, qubit_groups)
        arity, n_kraus, kraus = _ch_marshal(chans)
        nc = len(chans)
        if draws is None:
            draws = (rng if rng is not None else np.random.default_rng()).random(nc)
        r = np.ascontiguousarray(np.asarray(draws, dtype=np.float64).reshape(-1))
        if r.shape[0] != nc:
            raise ValueError("apply_kraus_channels: %d channels need %d draws, got %d" % (nc, nc, r.shape[0]))
        chosen = np.zeros(max(1, nc), dtype=np.uint32)
        cond = np.zeros(max(1, nc), dtype=np.float64)
        prob = C.c_double()
        self._chk(_lib.lib().qipb200_state_apply_kraus_channels(
            self._h, nc, _ptr(arity) if nc else None, _ptr(qa) if nc else None, _ptr(n_kraus) if nc else None,
            _ptr(kraus) if nc else None, _ptr(r) if nc else None, _ptr(chosen), _ptr(cond), C.byref(prob)))
        return chosen[:nc], cond[:nc], float(prob.value)

    def apply_function(self, fn: "Function", in_qubits: Sequence[int], out_qubits: Sequence[int] = ()):
        """Apply U|x>|y> = e^{i theta(x)} |x>|y XOR f(x)> of ``fn`` on the device: bit i of x is the value of qubit
        ``in_qubits[i]`` and bit i of f(x) is XORed into qubit ``out_qubits[i]`` (the convention of
        ``measure_probs``).

        One read-write sweep of the state in one kernel, in place (``function_plan`` gives the path).  Without theta
        the op only moves amplitudes and is exact.  Stream-ordered like ``apply_schedule``."""
        ia = np.ascontiguousarray(np.asarray(list(in_qubits), dtype=np.uint64))
        oa = np.ascontiguousarray(np.asarray(list(out_qubits), dtype=np.uint64))
        if ia.shape[0] != fn.n_in or oa.shape[0] != fn.n_out:
            raise ValueError("apply_function: the function takes %d input and %d output qubits, got %d and %d" % (
                fn.n_in, fn.n_out, ia.shape[0], oa.shape[0]))
        self._chk(_lib.lib().qipb200_state_apply_function(self._h, fn.handle, _ptr(ia) if ia.shape[0] else None,
                                                          _ptr(oa) if oa.shape[0] else None))

    def expect_function(self, fn: "Function", in_qubits: Sequence[int]) -> float:
        """<psi|D|psi> = sum_j |psi_j|^2 theta(x(j), p) for D = diag theta of a code function made with
        ``theta=True`` (e.g. the QAOA energy <C> of a cost C), on the state as it is (not renormalised), computed on
        the device in one read sweep; bit i of x is the value of qubit ``in_qubits[i]``.  Accumulated in double in a
        fixed order (bit-identical on repeated calls); synchronises."""
        ia = np.ascontiguousarray(np.asarray(list(in_qubits), dtype=np.uint64))
        if ia.shape[0] != fn.n_in:
            raise ValueError("expect_function: the function takes %d input qubits, got %d" % (fn.n_in, ia.shape[0]))
        out = C.c_double()
        self._chk(_lib.lib().qipb200_state_expect_function(self._h, fn.handle, _ptr(ia), C.byref(out)))
        return float(out.value)

    def apply_pauli_sum(self, src: "State", terms, coeffs):
        """Set this state to H|src> for H = sum_h coeffs[h] P_h, a real Pauli sum, on the device (out of place).

        Terms are encoded as for ``expect_paulis``; an empty term is the identity, and no terms give zero.  ``src``
        must be another state of the same context, precision and size; its pending collapse is applied first and
        this state takes its qubit layout.  Deterministic; stream-ordered like ``apply_schedule``
        (``pauli_sum_plan`` gives the sweep count).  For example ``w.apply_pauli_sum(st, H, c)`` then ``w.norm2()``
        is <psi|H^2|psi>."""
        args = _pauli_args("apply_pauli_sum", terms, coeffs, "coefficients")
        self._chk(_lib.lib().qipb200_state_apply_pauli_sum(self._h, src._h, *args))

    def energy_gradient(self, work: "State", ansatz, angles, hamiltonian, coeffs):
        """Energy and gradient of E(angles) = <psi0|U^dagger H U|psi0> by the adjoint method, on the device.

        This state holds psi0 on entry; U applies exp(-i angles[t]/2 P_t) for the ``ansatz`` strings, term 0 first
        (as ``apply_pauli_rotations``), and H = sum_h coeffs[h] Q_h (as ``apply_pauli_sum``).  Returns (E, g) with
        g[t] = dE/dangles[t]; a parameter shared by several strings has the sum of their entries as its derivative.
        ``work`` is scratch of the same size and precision: it ends holding U^dagger H U psi0.  This state ends at
        psi0 up to rounding (run forward and back); re-prepare psi0 when it is needed exactly.  Deterministic;
        synchronises (``pauli_gradient_plan`` gives the sweep counts)."""
        a = _pauli_args("energy_gradient", ansatz, angles, "angles")
        h = _pauli_args("energy_gradient", hamiltonian, coeffs, "coefficients", kind="Hamiltonian terms")
        T = a[3]
        energy = np.zeros(1, dtype=np.float64)
        grad = np.zeros(max(1, T), dtype=np.float64)
        self._chk(_lib.lib().qipb200_state_pauli_energy_gradient(self._h, work._h, *a, *h, _ptr(energy), _ptr(grad)))
        return float(energy[0]), grad[:T]

    def geometric_tensor(self, work_a: "State", work_b: "State", ansatz, angles):
        """The quantum geometric tensor of the Pauli-rotation circuit U = R_{T-1} ... R_0, R_t = exp(-i angles[t]/2 P_t)
        (``ansatz`` encoded as for ``apply_pauli_rotations``), at the state on entry psi0, on the device.

        Returns (G, e): G is a complex128 (T, T) array with G_ij = <d_i psi|d_j psi> - <d_i psi|psi><psi|d_j psi>
        for psi = U psi0, exactly Hermitian; e[t] = <psi_t|P_t|psi_t> (float64, (T,)), the expectation of P_t just
        before R_t.  Re G is the Fubini-Study metric: the matrix a quantum-natural-gradient step solves against
        (``np.linalg.lstsq(G.real, g)`` with g from ``energy_gradient``) and the A of McLachlan's imaginary-time
        equation A theta' = -grad E.  4 Re G is the quantum Fisher information, and Im G is the antisymmetric term of
        variational real-time evolution.  A parameter shared by several strings (one QAOA angle on many strings) gets
        A^T G A for its term-to-parameter matrix A (A[t, k] = 1 when string t carries parameter k), computed on the
        host.  ``work_a`` and ``work_b`` are two more states of the same context, precision and size, used as scratch;
        this state ends at U psi0, bit-identical to ``apply_pauli_rotations``.  Deterministic; synchronises; at most
        2048 terms (``pauli_geometric_tensor_plan`` gives the counts)."""
        args = _pauli_args("geometric_tensor", ansatz, angles, "angles")
        T = args[3]
        g = np.zeros(max(1, 2 * T * T), dtype=np.float64)
        e = np.zeros(max(1, T), dtype=np.float64)
        self._chk(_lib.lib().qipb200_state_pauli_geometric_tensor(self._h, work_a._h, work_b._h, *args, _ptr(g),
                                                                  _ptr(e)))
        return g[: 2 * T * T].view(np.complex128).reshape(T, T), e[:T]

    def evolve_pauli_sum(self, work_a: "State", work_b: "State", terms, coeffs, time: float, tol=None):
        """Set this state to exp(-i time H)|psi> for H = sum_h coeffs[h] P_h, a real Pauli sum, on the device.

        Terms are encoded as for ``apply_pauli_sum``.  A Chebyshev series in H~ = (H - a) / b (a: the identity terms'
        sum, b = sum |coeffs| of the others) is cut at the smallest degree K >= 2 whose tail bound tau_K is <= tol
        (default 1e-12 for complex128, 1e-6 for complex64); in exact arithmetic the result is then within
        tau_K |psi| of exp(-iHt)|psi>.  Returns (K, tau_K).  ``work_a`` and ``work_b`` are two more states of the same
        context, precision and size, used as scratch (their contents afterwards are unspecified).  Each of the K
        steps is one read-write sweep per sweep of ``pauli_sum_plan`` of the non-identity terms
        (``pauli_evolution_plan`` gives the counts); deterministic and stream-ordered.  K above 65536 is refused:
        split the time over several calls."""
        args = _pauli_args("evolve_pauli_sum", terms, coeffs, "coefficients")
        degree, tail = C.c_uint32(), C.c_double()
        self._chk(_lib.lib().qipb200_state_evolve_pauli_sum(
            self._h, work_a._h, work_b._h, *args, float(time),
            float(_default_tol(self.dtype) if tol is None else tol), C.byref(degree), C.byref(tail)))
        return int(degree.value), float(tail.value)

    def lanczos_pauli_sum(self, work_a: "State", work_b: "State", terms, coeffs, max_steps: int = 300, tol=None,
                          vector: bool = True) -> "LanczosResult":
        """The lowest eigenvalue of H = sum_h coeffs[h] P_h, a real Pauli sum, reachable from this state, by plain
        Lanczos on the device.

        Terms are encoded as for ``apply_pauli_sum``.  Runs from v_0 = psi / |psi| until the estimate
        rho_m = beta_m |y_(m-1)| of the m-step tridiagonal's lowest Ritz pair (theta, y) is <= tol b, b = sum |coeffs|
        of the non-identity terms (default tol 1e-8 for complex128, 1e-3 for complex64), or ``max_steps`` (<= 4096)
        steps: reaching the cap is not an error (``converged`` is False).  Only the part of the spectrum psi has weight
        on is reachable: a start state in a symmetry sector (fixed S_z, parity, ...) gives that sector's ground state.
        ``vector=False``: this state is not written, and (energy, residual) = (theta, rho_m).  ``vector=True``: a
        second pass rebuilds the same Lanczos vectors and this state ends as the normalised Ritz vector x / |x|;
        energy = <x|H|x> and residual = |Hx - energy x|, both computed on the device, and ``ritz_norm`` = |x| before
        normalisation (far from 1: loss of orthogonality).  In exact arithmetic some eigenvalue of H lies within
        residual of energy.  ``work_a`` and ``work_b`` are two more states of the same context, precision and size,
        used as scratch.  Deterministic; synchronises once per step (``pauli_lanczos_plan`` gives the kernel
        counts)."""
        args = _pauli_args("lanczos_pauli_sum", terms, coeffs, "coefficients")
        cap = max(1, min(int(max_steps), 4096))
        alpha, beta, out3 = np.zeros(cap), np.zeros(cap + 1), np.zeros(3)
        steps, conv = C.c_uint32(), C.c_uint32()
        self._chk(_lib.lib().qipb200_state_lanczos_pauli_sum(
            self._h, work_a._h, work_b._h, *args, int(max_steps),
            float(_default_lanczos_tol(self.dtype) if tol is None else tol), 1 if vector else 0, C.byref(steps),
            C.byref(conv), _ptr(alpha), _ptr(beta), _ptr(out3)))
        m = int(steps.value)
        return LanczosResult(float(out3[0]), float(out3[1]), m, bool(conv.value), alpha[:m].copy(),
                             beta[: m + 1].copy(), float(out3[2]))

    def reduced_density(self, qubits: Sequence[int]) -> np.ndarray:
        """Reduced density matrix of ``qubits`` (1 to 10 of them) on the state as it is (not renormalised), computed
        on the device: complex128 of shape (2^k, 2^k) with rho[a, b] = sum_r psi(r, a) conj(psi(r, b)).

        Bit i of the row and column indices a, b is the value of qubit ``qubits[i]`` (the convention of
        ``measure_probs``, so ``diag(rho)`` is ``measure_probs(qubits)`` up to rounding).  rho is exactly Hermitian
        and deterministic.  One read sweep of the state for k <= 6, 2^(k-6) sweeps above."""
        idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        k = len(idx)
        out = np.zeros((1 << min(k, 10)) ** 2 if k else 1, dtype=np.complex128)
        self._chk(_lib.lib().qipb200_state_reduced_density(self._h, _ptr(idx) if k else None, k, _ptr(out)))
        return out.reshape(1 << k, 1 << k)

    def _purity2(self, qubits):
        idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        out2 = np.zeros(2)
        self._chk(_lib.lib().qipb200_state_purity(self._h, _ptr(idx) if len(idx) else None, len(idx), _ptr(out2)))
        return float(out2[0]), float(out2[1])

    def purity(self, qubits: Sequence[int]) -> float:
        """Tr rho_A^2 = sum_{a,b} |rho_ab|^2 of the reduced density matrix of ``qubits`` on the state as it is (not
        renormalised: divide by ``norm2()**2`` for a state that is not a unit vector), computed on the device.

        The route depends on s = min(k, n - k): one norm2 sweep for k = n, ``reduced_density`` of the smaller side for
        s <= 10, and a Gram product on the FP64 tensor pipe above (``purity_plan`` reports it).  Deterministic."""
        return self._purity2(qubits)[0]

    def renyi2_entropy(self, qubits: Sequence[int]) -> float:
        """S_2 = -ln(Tr rho_A^2 / (Tr rho_A)^2) of ``qubits``: the Renyi-2 entanglement entropy across the cut, with
        the state normalised on the fly (one device call)."""
        p, tr = self._purity2(qubits)
        return -float(np.log(p / (tr * tr)))

    def _spectrum(self, qubits, rho):
        idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        k = len(idx)
        s = min(max(0, min(k, self.n - k)), 13)  # larger sides are refused by the call
        eigs = np.zeros(1 << s)
        out2 = np.zeros(2)
        r = np.zeros(1 << (2 * s), dtype=np.complex128) if rho else None
        _lib.preload_cusolver()
        self._chk(_lib.lib().qipb200_state_entanglement_spectrum(
            self._h, _ptr(idx) if k else None, k, _ptr(eigs), eigs.size, _ptr(r) if rho else None, _ptr(out2)))
        return eigs, (r.reshape(1 << s, 1 << s) if rho else None), float(out2[0]), float(out2[1])

    def entanglement_spectrum(self, qubits: Sequence[int], rho: bool = False):
        """Eigenvalues of the reduced density matrix across the cut between ``qubits`` and the rest, on the state as
        it is (not renormalised), in descending order: 2^s values for the smaller side of s = min(k, n - k) <= 13
        qubits.  They are the squared Schmidt coefficients times ``norm2()``, and the same whichever side is passed.

        With ``rho=True`` returns ``(eigs, rho)``, rho the side's 2^s x 2^s matrix (complex128) in the convention of
        ``reduced_density`` (which it equals for s <= 10); that needs k <= n - k, so that it is the matrix of the qubits
        passed.  The matrix is formed on the device (``reduced_density`` for s <= 10, the purity Gram kernel storing G
        for s = 11..13) and solved there by cuSOLVER; ``entanglement_spectrum_plan`` reports the route."""
        eigs, r, _, _ = self._spectrum(qubits, rho)
        return (eigs, r) if rho else eigs

    def entanglement_entropy(self, qubits: Sequence[int], alpha: float = 1.0) -> float:
        """Entanglement entropy across the cut, in nats, of the normalised spectrum p = lambda / Tr rho.  alpha = 1 is
        the von Neumann entropy -sum p ln p as the device call sums it; other alpha give the Renyi-alpha entropy
        ln(sum p^alpha) / (1 - alpha) from the spectrum, and alpha = inf the min-entropy -ln max p.  Eigenvalues that
        rounding left at or below 0 are dropped."""
        eigs, _, tr, h = self._spectrum(qubits, False)
        alpha = float(alpha)
        if alpha == 1.0:
            return h
        if tr == 0.0:
            return 0.0
        p = eigs[eigs > 0] / tr
        if np.isinf(alpha):
            return -float(np.log(p.max()))
        return float(np.log(np.sum(p ** alpha)) / (1.0 - alpha))

    # -- multi-GPU --------------------------------------------------------------
    def ipc_export(self):
        a = (C.c_ubyte * _lib.IPC_HANDLE_BYTES)()
        f = (C.c_ubyte * _lib.IPC_HANDLE_BYTES)()
        self._chk(_lib.lib().qipb200_state_ipc_export(self._h, a, f))
        return bytes(a), bytes(f)

    def ipc_import(self, amp_handles: bytes, flag_handles: bytes):
        assert len(amp_handles) == self.world_size * _lib.IPC_HANDLE_BYTES
        a = C.create_string_buffer(amp_handles, len(amp_handles))
        f = C.create_string_buffer(flag_handles, len(flag_handles))
        self._chk(_lib.lib().qipb200_state_ipc_import(self._h, a, f))

    def qubit_map(self):
        m = np.zeros(self.n, dtype=np.uint32)
        self._chk(_lib.lib().qipb200_state_qubit_map(self._h, _ptr(m)))
        return m

    def exchange_bytes(self) -> int:
        v = C.c_uint64()
        self._chk(_lib.lib().qipb200_state_exchange_bytes(self._h, C.byref(v)))
        return int(v.value)


class Function:
    """A classical function of an ``n_in``-qubit register kept on the device of ``ctx`` (qipb200_function), for
    ``State.apply_function``: U|x>|y> = e^{i theta(x)} |x>|y XOR f(x)>.

    ``f`` (n_out-bit integers) and ``theta`` (finite floats, radians) are arrays of length 2^n_in; ``f`` may be None
    when ``n_out`` is 0 (a phase oracle) and ``theta`` None for a pure permutation.  The table is checked and uploaded
    once, and the handle serves states of either precision on this context.  n_in <= 26, n_out <= 32."""

    def __init__(self, ctx: Context, n_in: int, n_out: int, f=None, theta=None):
        self.ctx, self.n_in, self.n_out = ctx, int(n_in), int(n_out)
        self._h = C.c_void_p()
        size = 1 << self.n_in if 1 <= self.n_in <= 26 else None  # other sizes are refused by the C entry
        fa = ta = None
        if f is not None:
            fa = np.ascontiguousarray(np.asarray(f, dtype=np.uint64).reshape(-1))
            if size is not None and fa.shape[0] != size:
                raise ValueError("Function: f has %d entries, 2^n_in = %d" % (fa.shape[0], size))
        if theta is not None:
            ta = np.ascontiguousarray(np.asarray(theta, dtype=np.float64).reshape(-1))
            if size is not None and ta.shape[0] != size:
                raise ValueError("Function: theta has %d entries, 2^n_in = %d" % (ta.shape[0], size))
        _lib.check(_lib.lib().qipb200_function_new(ctx.handle, self.n_in, self.n_out,
                                                   None if fa is None else _ptr(fa), None if ta is None else _ptr(ta),
                                                   C.byref(self._h)), ctx.handle)

    @classmethod
    def from_code(cls, ctx: Context, n_in: int, n_out: int, source: str, theta: bool = False,
                  n_params: int = 0) -> "Function":
        """A function given as CUDA source (qipb200_function_new_code), evaluated on the device: no table, so
        ``n_in`` may cover the whole state (n_in + n_out <= 34, n_out <= 32).

        ``source`` defines ``__device__ uint64_t qip_f(uint64_t x)`` when ``n_out > 0`` and, with ``theta=True``,
        ``__device__ double qip_theta(uint64_t x, const double *p)`` where ``p`` holds the ``n_params`` (<= 16)
        parameters of ``set_params`` (all 0 at first).  It is compiled with NVRTC for sm_90a (cached in the process
        and in ``QIPB200_JIT_CACHE_DIR``); a compile error raises ``CircuitError`` with the NVRTC log.  f is checked
        over every x (f(x) < 2^n_out) and theta with the zero parameters (finite) before the handle is returned."""
        self = cls.__new__(cls)
        self.ctx, self.n_in, self.n_out, self.n_params = ctx, int(n_in), int(n_out), int(n_params)
        self._h = C.c_void_p()
        log = C.create_string_buffer(1 << 16)
        _lib.check(_lib.lib().qipb200_function_new_code(ctx.handle, self.n_in, self.n_out, source.encode("utf-8"),
                                                        FN_CODE_THETA if theta else 0, self.n_params, log,
                                                        len(log), C.byref(self._h)), ctx.handle)
        return self

    def set_params(self, params):
        """Set the parameters theta(x, p) of a code function is evaluated with; theta is checked finite for every x
        first (a refused vector raises ``CircuitError`` and keeps the previous parameters).  Later applies use the
        new values; applies already queued keep theirs.  Synchronises."""
        pa = np.ascontiguousarray(np.asarray(params, dtype=np.float64).reshape(-1))
        _lib.check(_lib.lib().qipb200_function_set_params(self._h, _ptr(pa) if pa.shape[0] else None, pa.shape[0]),
                   self.ctx.handle)

    def tabulate(self, x0: int = 0, count: int = None):
        """(f, cs) for x in [x0, x0 + count), evaluated on the device by the functions the apply kernels use:
        f (uint64) and cs (float64, shape (count, 2)) = (cos theta(x), sin theta(x)) in double, which the apply rounds
        once to the state's precision.  Without a phase cs is (1, 0); without an out register f is 0."""
        if count is None:
            count = (1 << self.n_in) - int(x0)
        f = np.zeros(max(1, int(count)), dtype=np.uint64)
        cs = np.zeros((max(1, int(count)), 2), dtype=np.float64)
        _lib.check(_lib.lib().qipb200_function_tabulate(self._h, int(x0), int(count), _ptr(f), _ptr(cs)),
                   self.ctx.handle)
        return f[: int(count)], cs[: int(count)]

    @property
    def handle(self):
        return self._h

    def free(self):
        """Release the device tables (stream-ordered: safe straight after an apply); a code function waits for the
        context's stream, then unloads its program."""
        if self._h:
            _lib.lib().qipb200_function_free(self._h)
            self._h = C.c_void_p()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.free()

    def __del__(self):  # pragma: no cover
        try:
            self.free()
        except Exception:
            pass


FUNCTION_TILE, FUNCTION_PAIR = 0, 1
FN_CODE_THETA = 1  # QIPB200_FN_CODE_THETA


class DensityMatrix:
    """The exact mixed state of n qubits on the device, for noisy circuits (qipb200_density_*).

    It owns a ``State`` of 2n qubits (``.state``) that holds vec(rho): row qubit q is state qubit q, column qubit q is
    state qubit n + q, so rho[r, c] is amplitude r * 2^n + c and ``download()`` is the 2^n x 2^n matrix.  Gates and
    Kraus channels run interleaved in one fused schedule (``apply``); the readouts honour a permuted layout, work on
    rho as it is (not renormalised) and are deterministic, except the bits of ``spectrum``, which come from cuSOLVER.
    Unsharded states only."""

    def __init__(self, n: int, dtype=np.complex128, ctx: Optional[Context] = None):
        if int(n) < 1:
            raise ValueError("DensityMatrix: n must be at least 1, got %d" % int(n))
        self.n = int(n)
        self.state = State(2 * self.n, dtype, ctx)
        self.ctx, self.prec, self.dtype = self.state.ctx, self.state.prec, self.state.dtype

    def free(self):
        self.state.free()

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.free()

    def _chk(self, st):
        _lib.check(st, self.ctx.handle)

    def set_basis(self, i: int):
        """rho = |i><i| (pending, like State.set_basis: the next fused apply builds it in its first pass)."""
        i = int(i)
        if not 0 <= i < (1 << self.n):
            raise ValueError("set_basis: %d is not an index of %d qubits" % (i, self.n))
        self.state.set_basis(i + (i << self.n))

    def set_pure(self, psi: State):
        """rho = |psi><psi| (not normalised) for a State of n qubits in this context and precision: one write sweep."""
        self._chk(_lib.lib().qipb200_density_from_state(self.state._h, psi._h))

    def apply(self, items, fusion: bool = True):
        """Run ``items`` in order in one schedule: each is a ``MatrixOp`` (rho -> U rho U^dagger) or a pair
        ``(channel, qubits)`` with a ``channels.KrausChannel`` or ``Channel`` on 1..4 qubits (rho -> sum K rho
        K^dagger, the channel's first qubit the most significant bit of its matrices).  ``fusion`` as for
        ``State.apply_schedule``; the result is bit-identical to ``state.apply_schedule(density_schedule(...))`` when both
        run the same kernels (QIPB200_JIT: a pass may run on the interpreter kernel while its generated kernel
        compiles)."""
        args, keep = _density_args(self.prec, items)
        flags = _lib.SCHED_DEFAULT if fusion else _lib.SCHED_NO_FUSION
        self._chk(_lib.lib().qipb200_density_apply(self.state._h, *args, flags))

    def measure_probs(self, qubits: Sequence[int]) -> np.ndarray:
        """out[m] = sum of rho_rr over the r whose bits on ``qubits`` equal m (bit i of m is qubits[i]); reads only the
        diagonal.  No qubits gives [Tr rho]."""
        idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        out = np.zeros(1 << len(idx), dtype=np.float64)
        self._chk(_lib.lib().qipb200_density_measure_probs(self.state._h, _ptr(idx) if len(idx) else None, len(idx),
                                                           _ptr(out)))
        return out

    def trace(self) -> float:
        return float(self.measure_probs([])[0])

    def sample(self, qubits: Sequence[int], shots: int, rng=None) -> np.ndarray:
        """``shots`` outcomes of measuring ``qubits`` (bit i of each is qubits[i]), drawn on the host from
        ``measure_probs`` (at most 2^n values) with ``rng`` (a fresh ``np.random.default_rng()`` when None)."""
        p = np.clip(self.measure_probs(qubits), 0.0, None)
        rng = rng if rng is not None else np.random.default_rng()
        return rng.choice(p.shape[0], size=int(shots), p=p / p.sum()).astype(np.uint64)

    def measure(self, qubits: Sequence[int], rng=None):
        """Selective measurement of ``qubits``: draws the outcome m with probability p = measure_probs(qubits)[m] and
        leaves rho = Pi rho Pi / p.  Pi is applied as one single-qubit projector per measured qubit through ``apply``,
        the first scaled by 1/sqrt(p).  Returns (m, p)."""
        qubits = [int(q) for q in qubits]
        probs = np.clip(self.measure_probs(qubits), 0.0, None)
        total = float(probs.sum())
        if not total > 0.0:
            raise CircuitError("measure: the density matrix has no weight on these qubits")
        u = (rng if rng is not None else np.random.default_rng()).random() * total
        m = int(min(np.searchsorted(np.cumsum(probs), u, side="right"), probs.shape[0] - 1))
        while probs[m] == 0.0:  # rounding at the end of the cumulative sum
            m -= 1
        p = float(probs[m])
        ops = []
        for j, q in enumerate(qubits):
            proj = np.zeros((2, 2), dtype=np.complex128)
            proj[(m >> j) & 1, (m >> j) & 1] = 1.0 / np.sqrt(p) if j == 0 else 1.0
            ops.append(MatrixOp.new_matrix([q], proj.reshape(-1)))
        self.apply(ops)
        return m, p

    def expect_paulis(self, terms) -> np.ndarray:
        """Re Tr(rho P_t) for Pauli strings encoded as for ``State.expect_paulis``."""
        qs, ls, lens = _marshal_paulis(terms)
        out = np.zeros(max(1, lens.shape[0]), dtype=np.float64)
        self._chk(_lib.lib().qipb200_density_expect_paulis(self.state._h, _ptr(qs), ls, _ptr(lens), lens.shape[0],
                                                           _ptr(out)))
        return out[: lens.shape[0]]

    def reduced_density(self, qubits: Sequence[int]) -> np.ndarray:
        """Tr_B rho for 1..10 kept ``qubits``: complex128 (2^k, 2^k), bit i of the indices qubits[i] (the convention
        of ``State.reduced_density``); exactly Hermitian."""
        idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
        k = len(idx)
        out = np.zeros((1 << min(k, 10)) ** 2 if k else 1, dtype=np.complex128)
        self._chk(_lib.lib().qipb200_density_reduced(self.state._h, _ptr(idx) if k else None, k, _ptr(out)))
        return out.reshape(1 << k, 1 << k)

    def fidelity(self, psi: State) -> float:
        """<psi|rho|psi> for a State of n qubits (its real part; the imaginary part is rounding only): one read sweep
        of rho."""
        out2 = np.zeros(2)
        self._chk(_lib.lib().qipb200_density_fidelity(self.state._h, psi._h, _ptr(out2)))
        return float(out2[0])

    def purity(self) -> float:
        """Tr rho^2 = sum |rho_rc|^2: ``norm2`` of the vector."""
        return self.state.norm2()

    def spectrum(self) -> np.ndarray:
        """The 2^n eigenvalues of rho in descending order (n <= 13), solved on the device by cuSOLVER."""
        eigs = np.zeros(1 << min(self.n, 13))
        _lib.preload_cusolver()
        self._chk(_lib.lib().qipb200_density_spectrum(self.state._h, _ptr(eigs)))
        return eigs

    def entropy(self) -> float:
        """von Neumann entropy -sum p ln p in nats of p = lambda / Tr rho over the eigenvalues > 0."""
        eigs = self.spectrum()
        tr = self.trace()
        p = eigs[eigs > 0] / tr
        return float(-np.sum(p * np.log(p)))

    def download(self) -> np.ndarray:
        side = 1 << self.n
        return self.state.download().reshape(side, side)


def _density_args(prec, items):
    """((ops, n_ops, n_channels, channel_pos, arity, qubits, n_kraus, kraus), keep): the C arguments of a list of
    MatrixOps and (channel, qubits) pairs, and the arrays they point into (hold keep for the call)."""
    from . import channels as _ch
    ops, chans, groups, pos = [], [], [], []
    for item in items:
        if isinstance(item, MatrixOp):
            ops.append(item)
            continue
        chan, qs = item
        chan = chan if isinstance(chan, _ch.KrausChannel) else _ch.KrausChannel(chan)
        qs = [int(q) for q in qs]
        if chan.n_qubits != len(qs):
            raise ValueError("density: channel %d acts on %d qubits but is given %d" % (len(chans), chan.n_qubits,
                                                                                    len(qs)))
        chans.append(chan)
        groups.append(qs)
        pos.append(len(ops))
    arr, keep = marshal_ops(ops, prec)
    arity, n_kraus, kraus = _ch_marshal(chans)
    qa = np.ascontiguousarray(np.asarray([q for g in groups for q in g], dtype=np.uint64))
    cp = np.ascontiguousarray(np.asarray(pos, dtype=np.uint64))
    nc = len(chans)
    args = (arr, len(ops), nc, _ptr(cp) if nc else None, _ptr(arity) if nc else None, _ptr(qa) if nc else None,
            _ptr(n_kraus) if nc else None, _ptr(kraus) if nc else None)
    return args, (keep, arity, n_kraus, kraus, qa, cp)


def density_schedule(n: int, dtype, items):
    """The doubled schedule of ``DensityMatrix.apply(items)`` on an n-qubit rho, as MatrixOps on 2n qubits, written by
    the library (qipb200_density_schedule, QIPS v1) and decoded here; needs no GPU.  Validates as the call does."""
    from .wire import loads_schedule
    prec = prec_of(dtype)
    args, keep = _density_args(prec, items)
    need = C.c_size_t(0)
    L = _lib.lib()
    st = L.qipb200_density_schedule(prec, int(n), *args, None, 0, C.byref(need))
    if st != _lib.ERR_SIZE_MISMATCH or need.value == 0:
        _lib.check(st, None)
    buf = (C.c_ubyte * need.value)()
    _lib.check(L.qipb200_density_schedule(prec, int(n), *args, buf, need.value, C.byref(need)), None)
    _, _, ops = loads_schedule(bytes(buf))
    return ops


def function_code_compile(n_in: int, n_out: int, source: str, theta: bool = False, n_params: int = 0) -> str:
    """Compile the program of ``Function.from_code`` with NVRTC without a context or GPU; returns the NVRTC log
    (warnings, if any) and raises ``CircuitError`` (with the log) on a compile error or refused sizes."""
    log = C.create_string_buffer(1 << 16)
    _lib.check(_lib.lib().qipb200_function_code_compile(int(n_in), int(n_out), source.encode("utf-8"),
                                                        FN_CODE_THETA if theta else 0, int(n_params), log, len(log)),
               None)
    return log.value.decode("utf-8", "replace")


def function_plan(n: int, dtype, in_qubits: Sequence[int], out_qubits: Sequence[int] = ()):
    """(path, tile bits) of State.apply_function on an unsharded n-qubit state in canonical layout (needs no GPU):
    path FUNCTION_TILE (0, the staged tile path) or FUNCTION_PAIR (1, tile bits 0)."""
    ia = np.ascontiguousarray(np.asarray(list(in_qubits), dtype=np.uint64))
    oa = np.ascontiguousarray(np.asarray(list(out_qubits), dtype=np.uint64))
    v = (C.c_uint32 * 2)()
    _lib.check(_lib.lib().qipb200_function_plan(prec_of(dtype), int(n), _ptr(ia) if ia.shape[0] else None,
                                                ia.shape[0], _ptr(oa) if oa.shape[0] else None, oa.shape[0], v), None)
    return int(v[0]), int(v[1])


def channels_plan(n: int, dtype, channels, qubits: Sequence[int]):
    """(state-dependent channels, read sweeps at most, read-write sweeps at most, kernels at most) of
    State.apply_channels on an unsharded n-qubit state with nothing pending (needs no GPU); validates as the call
    does."""
    from . import channels as _ch
    qa = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
    chans = [channels] * qa.shape[0] if isinstance(channels, _ch.Channel) else list(channels)
    if len(chans) != qa.shape[0]:
        raise ValueError("channels_plan: %d channels but %d qubits" % (len(chans), qa.shape[0]))
    _single_qubit("channels_plan", chans, "multiqubit_channels_plan")
    _, n_kraus, kraus = _ch.marshal(chans)
    v = (C.c_uint32 * 4)()
    k = qa.shape[0]
    _lib.check(_lib.lib().qipb200_channels_plan(prec_of(dtype), int(n), k, _ptr(qa) if k else None,
                                                _ptr(n_kraus) if k else None, _ptr(kraus) if k else None, v), None)
    return tuple(int(x) for x in v)


def _ch_marshal(chans):
    from . import channels as _ch
    return _ch.marshal(chans)


def _single_qubit(who, chans, instead):
    for c, chan in enumerate(chans):
        if chan.n_qubits != 1:
            raise ValueError("%s: channel %d acts on %d qubits; use %s" % (who, c, chan.n_qubits, instead))


def _channel_groups(who, channels, qubit_groups):
    """(channels, flat uint64 qubits) of a multi-qubit layer; one Channel stands for every group."""
    from . import channels as _ch
    groups = [[int(q) for q in g] for g in qubit_groups]
    chans = [channels] * len(groups) if isinstance(channels, _ch.Channel) else list(channels)
    if len(chans) != len(groups):
        raise ValueError("%s: %d channels but %d qubit groups" % (who, len(chans), len(groups)))
    for c, (chan, g) in enumerate(zip(chans, groups)):
        if chan.n_qubits != len(g):
            raise ValueError("%s: channel %d acts on %d qubits but its group has %d" % (who, c, chan.n_qubits, len(g)))
    qa = np.ascontiguousarray(np.asarray([q for g in groups for q in g], dtype=np.uint64))
    return chans, qa


def multiqubit_channels_plan(n: int, dtype, channels, qubit_groups):
    """(state-dependent channels, read sweeps at most, read-write sweeps at most, kernels at most) of
    State.apply_multiqubit_channels on an unsharded n-qubit state with nothing pending (needs no GPU); validates as
    the call does."""
    chans, qa = _channel_groups("multiqubit_channels_plan", channels, qubit_groups)
    arity, n_kraus, kraus = _ch_marshal(chans)
    v = (C.c_uint32 * 4)()
    k = len(chans)
    _lib.check(_lib.lib().qipb200_multiqubit_channels_plan(
        prec_of(dtype), int(n), k, _ptr(arity) if k else None, _ptr(qa) if k else None,
        _ptr(n_kraus) if k else None, _ptr(kraus) if k else None, v), None)
    return tuple(int(x) for x in v)


def _kraus_groups(who, channels, qubit_groups):
    """(KrausChannels, flat uint64 qubits) of a Kraus layer; one channel stands for every group, and a Channel is
    taken as the KrausChannel of its operators."""
    from . import channels as _ch
    qubit_groups = [list(g) for g in qubit_groups]
    one = isinstance(channels, (_ch.Channel, _ch.KrausChannel))
    chans = [channels] * len(qubit_groups) if one else list(channels)
    chans = [c if isinstance(c, _ch.KrausChannel) else _ch.KrausChannel(c) for c in chans]
    return _channel_groups(who, chans, qubit_groups)


def kraus_channels_plan(n: int, dtype, channels, qubit_groups):
    """(groups r, read sweeps, read-write sweeps, kernels) of State.apply_kraus_channels on an unsharded n-qubit state
    with nothing pending (needs no GPU); the state-independent channels' schedule is not counted.  Validates as the
    call does."""
    chans, qa = _kraus_groups("kraus_channels_plan", channels, qubit_groups)
    arity, n_kraus, kraus = _ch_marshal(chans)
    v = (C.c_uint32 * 4)()
    k = len(chans)
    _lib.check(_lib.lib().qipb200_kraus_channels_plan(
        prec_of(dtype), int(n), k, _ptr(arity) if k else None, _ptr(qa) if k else None,
        _ptr(n_kraus) if k else None, _ptr(kraus) if k else None, v), None)
    return tuple(int(x) for x in v)


def validate_op(op: MatrixOp, n: int, dtype=np.complex128):
    """make_*_op checks + index range at the ABI; needs no GPU."""
    prec = prec_of(dtype)
    cop, keep = marshal_op(op, prec)
    _lib.check(_lib.lib().qipb200_validate_op(None, prec, int(n), C.byref(cop)), None)


def _marshal_paulis(terms):
    """Flat (qubits u64, letters bytes, term lengths u32) arrays of the C ABI from [[(letter, qubit), ...], ...]."""
    qs, ls, lens = [], [], []
    for t in terms:
        t = list(t)
        lens.append(len(t))
        for letter, q in t:
            b = letter.encode("ascii") if isinstance(letter, str) else bytes(letter)
            if len(b) != 1:
                raise ValueError("Pauli letter must be one character, got %r" % (letter,))
            ls.append(b)
            qs.append(int(q))
    qa = np.ascontiguousarray(np.asarray(qs if qs else [0], dtype=np.uint64))
    la = C.create_string_buffer(b"".join(ls) or b"\0", max(1, len(ls)))
    return qa, la, np.ascontiguousarray(np.asarray(lens if lens else [0], dtype=np.uint32))[: len(lens)]


def _pauli_term_args(terms):
    """(qubits, letters, term lengths, term count) C arguments of a term list; the pointers keep their arrays alive."""
    qs, ls, lens = _marshal_paulis(terms)
    return qs.ctypes.data_as(C.c_void_p), ls, lens.ctypes.data_as(C.c_void_p), lens.shape[0]


def _pauli_args(who, terms, values, what, kind="terms"):
    """The C arguments of a term list followed by its values (float64, one per term; NULL for no terms)."""
    v = np.ascontiguousarray(np.asarray(values, dtype=np.float64).reshape(-1))
    terms = list(terms)
    if v.shape[0] != len(terms):
        raise ValueError("%s: %d %s but %d %s" % (who, len(terms), kind, v.shape[0], what))
    return _pauli_term_args(terms) + (v.ctypes.data_as(C.c_void_p) if v.shape[0] else None,)


def _pauli_plan(entry, n, dtype, count, *term_lists):
    """The count uint32 results of the host-only plan qipb200_<entry> of these term lists."""
    v = (C.c_uint32 * count)()
    args = [a for terms in term_lists for a in _pauli_term_args(terms)]
    _lib.check(getattr(_lib.lib(), "qipb200_" + entry)(prec_of(dtype), int(n), *args, v), None)
    return tuple(int(x) for x in v)


def expect_plan(n: int, dtype, terms) -> int:
    """Read sweeps State.expect_paulis makes for these terms on an unsharded n-qubit state (needs no GPU)."""
    return _pauli_plan("expect_plan", n, dtype, 1, terms)[0]


def transition_plan(n: int, dtype, terms):
    """(read sweeps, kernels) of State.transition_paulis for these terms on unsharded n-qubit states in canonical
    layout with nothing pending (needs no GPU); (0, 0) for no terms."""
    return _pauli_plan("transition_plan", n, dtype, 2, terms)


def purity_plan(n: int, dtype, qubits):
    """(route, s, kernels, Gram blocks) of State.purity for these qubits on an unsharded n-qubit state (needs no GPU):
    route 0 is norm2 (k = n), 1 reduced_density (s <= 10), 2 the Gram kernel; s = min(k, n - k)."""
    idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
    v = (C.c_uint32 * 4)()
    _lib.check(_lib.lib().qipb200_purity_plan(prec_of(dtype), int(n), _ptr(idx) if len(idx) else None, len(idx), v),
               None)
    return tuple(int(x) for x in v)


def entanglement_spectrum_plan(n: int, dtype, qubits):
    """(route, s, kernels, device matrix bytes, solver loads) of State.entanglement_spectrum for these qubits on an
    unsharded n-qubit state (needs no GPU): the routes of purity_plan, with route 2 one Gram kernel that stores G;
    the last field is 1 when cuSOLVER loads in this process."""
    idx = np.ascontiguousarray(np.asarray(list(qubits), dtype=np.uint64))
    v = (C.c_uint32 * 5)()
    _lib.preload_cusolver()
    _lib.check(_lib.lib().qipb200_entanglement_spectrum_plan(prec_of(dtype), int(n), _ptr(idx) if len(idx) else None,
                                                            len(idx), v), None)
    return tuple(int(x) for x in v)


def pauli_rotation_plan(n: int, dtype, terms) -> int:
    """Read-write sweeps State.apply_pauli_rotations makes for these terms on an unsharded n-qubit state (needs no
    GPU)."""
    return _pauli_plan("pauli_rotation_plan", n, dtype, 1, terms)[0]


def pauli_sum_plan(n: int, dtype, terms) -> int:
    """Read-write sweeps State.apply_pauli_sum makes for these terms on an unsharded n-qubit state (needs no GPU)."""
    return _pauli_plan("pauli_sum_plan", n, dtype, 1, terms)[0]


def pauli_gradient_plan(n: int, dtype, ansatz, hamiltonian):
    """(forward, sum, backward) sweeps State.energy_gradient makes on an unsharded n-qubit state (needs no GPU); the
    call launches forward + sum + 2 * backward kernels."""
    return _pauli_plan("pauli_gradient_plan", n, dtype, 3, ansatz, hamiltonian)


def pauli_geometric_tensor_plan(n: int, dtype, ansatz):
    """(forks, segment sweeps, kernels) of State.geometric_tensor on an unsharded n-qubit state (needs no GPU): one
    fork per term, the sweeps of terms i+1 .. T-1 summed over i, and T + 2 sweeps + 1 kernels (0 for no terms)."""
    return _pauli_plan("pauli_geometric_tensor_plan", n, dtype, 3, ansatz)


def _default_tol(dtype):
    return 1e-12 if np.dtype(cdtype(prec_of(dtype))) == np.complex128 else 1e-6


def pauli_evolution_plan(n: int, dtype, terms, coeffs, time: float, tol=None):
    """(degree, sweeps per step, kernels, tail, C) of State.evolve_pauli_sum on an unsharded n-qubit state (needs no
    GPU): C[k] (complex128, K + 1 of them) are the series coefficients (2 - delta_k0) (-i)^k J_k(bt) e^{-iat}."""
    args = _pauli_args("pauli_evolution_plan", terms, coeffs, "coefficients")
    tol = float(_default_tol(dtype) if tol is None else tol)
    v, tail = (C.c_uint32 * 3)(), C.c_double()

    def call(out, cap):
        _lib.check(_lib.lib().qipb200_pauli_evolution_plan(prec_of(dtype), int(n), *args, float(time), tol, v,
                                                           C.byref(tail), out, cap), None)

    call(None, 0)
    out = np.zeros(2 * (int(v[0]) + 1), dtype=np.float64)
    call(_ptr(out), out.shape[0])
    return int(v[0]), int(v[1]), int(v[2]), float(tail.value), out.view(np.complex128)


class LanczosResult(NamedTuple):
    """What State.lanczos_pauli_sum returns: alpha[0..steps), beta[0..steps] (beta[0] = |psi|)."""
    energy: float
    residual: float
    steps: int
    converged: bool
    alpha: np.ndarray
    beta: np.ndarray
    ritz_norm: float


def _default_lanczos_tol(dtype):
    return 1e-8 if np.dtype(cdtype(prec_of(dtype))) == np.complex128 else 1e-3


def pauli_lanczos_plan(n: int, dtype, terms):
    """(sum sweeps per step, kernels per first-pass step, kernels per second-pass step, kernels outside the steps in
    vector mode) of State.lanczos_pauli_sum on an unsharded n-qubit state (needs no GPU).  A call of m steps launches
    1 + m k1 kernels without the vector, m k1 + (m - 1) k2 + k0 with it; (0, 0, 0, 2) when every term is the
    identity."""
    return _pauli_plan("pauli_lanczos_plan", n, dtype, 4, terms)


def lanczos_ritz(alpha, beta):
    """(theta, y, estimate) for the tridiagonal of alpha[0..m) and beta[0..m] as State.lanczos_pauli_sum returns them:
    the lowest eigenvalue theta of T_m (off-diagonal beta[1..m)), its unit eigenvector y (y[0] >= 0) and
    beta[m] |y[m-1]| -- the solve the call runs after every step (needs no GPU)."""
    a = np.ascontiguousarray(np.asarray(alpha, dtype=np.float64).reshape(-1))
    b = np.ascontiguousarray(np.asarray(beta, dtype=np.float64).reshape(-1))
    m = a.shape[0]
    if b.shape[0] != m + 1:
        raise ValueError("lanczos_ritz: %d alphas need %d betas, got %d" % (m, m + 1, b.shape[0]))
    theta, est = C.c_double(), C.c_double()
    y = np.zeros(max(1, m))
    _lib.check(_lib.lib().qipb200_lanczos_ritz(_ptr(a) if m else None, _ptr(b), m, C.byref(theta), _ptr(y),
                                               C.byref(est)), None)
    return float(theta.value), y[:m], float(est.value)


def plan_exchanges(ops: Sequence[MatrixOp], n: int, world_size: int, dtype=np.complex128):
    prec = prec_of(dtype)
    arr, keep = marshal_ops(ops, prec)
    out = np.zeros(max(1, len(ops)), dtype=np.uint32)
    _lib.check(_lib.lib().qipb200_plan_exchanges(prec, int(n), int(world_size), arr, len(ops), _ptr(out)), None)
    return out[: len(ops)]
