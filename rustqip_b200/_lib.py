"""Loader + ctypes signatures of rustqip_b200/libqipb200.so (include/qipb200.h).

The product path fails loudly when the CUDA extension is missing: there is no
CPU fallback anywhere in this package.
"""
from __future__ import annotations

import ctypes as C
import os

from ._abi import QipOp
from .errors import B200Unavailable, CircuitError

_HERE = os.path.dirname(os.path.abspath(__file__))
SO_PATH = os.environ.get("QIPB200_LIB") or os.path.join(_HERE, "libqipb200.so")  # QIPB200_LIB: a development build
IPC_HANDLE_BYTES = 64

SCHED_DEFAULT = 0
SCHED_NO_FUSION = 1
MEASURE_FORCED = 1
MEASURE_FORCED_PROB = 2
ERR_SIZE_MISMATCH = 2

_lib = None

# every symbol include/qipb200.h declares
EXPORTS = [
    "qipb200_abi_version", "qipb200_init", "qipb200_init_multi", "qipb200_shutdown", "qipb200_last_error",
    "qipb200_kernel_launches", "qipb200_launch_stats", "qipb200_kernel_counts", "qipb200_release_pool", "qipb200_stream_handle", "qipb200_jit_stats", "qipb200_jit_precompile", "qipb200_profile_enable", "qipb200_profile_read", "qipb200_validate_op", "qipb200_apply_op",
    "qipb200_apply_op_overwrite", "qipb200_apply_ops", "qipb200_state_new", "qipb200_state_free",
    "qipb200_state_set_basis", "qipb200_state_upload", "qipb200_state_download",
    "qipb200_state_apply_op", "qipb200_state_apply_schedule", "qipb200_state_norm2",
    "qipb200_state_sync", "qipb200_state_max_abs_diff", "qipb200_calculate_state", "qipb200_state_measure_probs",
    "qipb200_state_measure_prob", "qipb200_state_soft_measure", "qipb200_state_sample", "qipb200_state_collapse",
    "qipb200_state_measure", "qipb200_state_expect_paulis", "qipb200_expect_plan", "qipb200_state_transition_paulis",
    "qipb200_transition_plan", "qipb200_state_reduced_density", "qipb200_state_purity", "qipb200_purity_plan",
    "qipb200_state_entanglement_spectrum", "qipb200_entanglement_spectrum_plan",
    "qipb200_state_apply_pauli_rotations", "qipb200_pauli_rotation_plan", "qipb200_state_apply_channels",
    "qipb200_channels_plan", "qipb200_state_apply_multiqubit_channels", "qipb200_multiqubit_channels_plan",
    "qipb200_state_apply_kraus_channels", "qipb200_kraus_channels_plan",
    "qipb200_density_apply", "qipb200_density_schedule", "qipb200_density_from_state", "qipb200_density_measure_probs",
    "qipb200_density_expect_paulis", "qipb200_density_reduced", "qipb200_density_fidelity", "qipb200_density_spectrum",
    "qipb200_function_new",
    "qipb200_function_free", "qipb200_state_apply_function", "qipb200_function_plan", "qipb200_function_new_code",
    "qipb200_function_set_params", "qipb200_function_code_compile", "qipb200_function_tabulate",
    "qipb200_state_expect_function", "qipb200_state_apply_pauli_sum",
    "qipb200_pauli_sum_plan", "qipb200_state_pauli_energy_gradient", "qipb200_pauli_gradient_plan",
    "qipb200_state_pauli_geometric_tensor", "qipb200_pauli_geometric_tensor_plan",
    "qipb200_state_evolve_pauli_sum", "qipb200_pauli_evolution_plan", "qipb200_state_lanczos_pauli_sum",
    "qipb200_pauli_lanczos_plan", "qipb200_lanczos_ritz",
    "qipb200_state_new_sharded", "qipb200_state_ipc_export", "qipb200_state_ipc_import",
    "qipb200_state_qubit_map", "qipb200_state_exchange_bytes", "qipb200_plan_exchanges",
    "qipb200_state_save", "qipb200_state_load", "qipb200_schedule_parse", "qipb200_schedule_ops", "qipb200_schedule_free", "qipb200_schedule_serialise",
]


_cusolver_checked = False


def preload_cusolver():
    """Optional, once per process, before the first entanglement-spectrum call: the library loads cuSOLVER with dlopen
    (libcusolver.so.11 on the loader path, then the CUDA toolkit's lib64).  Where neither exists, the copy that ships
    with the torch wheel (the nvidia-cusolver-cu12 package) is loaded here with RTLD_GLOBAL, its dependencies first, so
    that the library's dlopen finds it by name.  Nothing else depends on it; QIPB200_NO_CUSOLVER_PRELOAD=1 skips it."""
    global _cusolver_checked
    if _cusolver_checked or os.environ.get("QIPB200_NO_CUSOLVER_PRELOAD") == "1":
        return
    _cusolver_checked = True
    for name in ("libcusolver.so.11", "/usr/local/cuda/lib64/libcusolver.so.11"):
        try:
            C.CDLL(name)
            return
        except OSError:
            pass
    try:
        import nvidia  # the namespace package of the CUDA wheels torch depends on
    except ImportError:
        return
    for base in nvidia.__path__:
        for pkg, so in (("nvjitlink", "libnvJitLink.so.12"), ("cublas", "libcublasLt.so.12"),
                        ("cublas", "libcublas.so.12"), ("cusparse", "libcusparse.so.12"),
                        ("cusolver", "libcusolver.so.11")):
            path = os.path.join(base, pkg, "lib", so)
            if os.path.exists(path):
                try:
                    C.CDLL(path, mode=C.RTLD_GLOBAL)
                except OSError:
                    return


def lib():
    """Load libqipb200.so (built in-tree by `make -C rustqip_b200/csrc` / __graft_entry__.build())."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(SO_PATH):
        raise B200Unavailable(
            "%s is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(nvcc, sm_90a). rustqip_b200 has no CPU fallback." % SO_PATH)
    L = C.CDLL(SO_PATH)
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
    opp = C.POINTER(QipOp)
    L.qipb200_abi_version.restype = i32
    L.qipb200_init.restype, L.qipb200_init.argtypes = i32, [C.POINTER(vp), i32]
    L.qipb200_init_multi.restype, L.qipb200_init_multi.argtypes = i32, [C.POINTER(vp), i32, vp]
    L.qipb200_shutdown.restype, L.qipb200_shutdown.argtypes = None, [vp]
    L.qipb200_last_error.restype, L.qipb200_last_error.argtypes = C.c_char_p, [vp]
    L.qipb200_stream_handle.restype, L.qipb200_stream_handle.argtypes = i32, [vp, C.POINTER(vp)]
    L.qipb200_launch_stats.restype, L.qipb200_launch_stats.argtypes = i32, [vp, vp]
    L.qipb200_jit_stats.restype = i32
    L.qipb200_jit_stats.argtypes = [vp, i32, vp, C.c_char_p, C.c_size_t]
    L.qipb200_jit_precompile.restype = i32
    L.qipb200_jit_precompile.argtypes = [i32, u32, opp, C.c_size_t, vp, C.c_char_p, C.c_size_t]
    L.qipb200_profile_enable.restype, L.qipb200_profile_enable.argtypes = i32, [vp, i32]
    L.qipb200_profile_read.restype, L.qipb200_profile_read.argtypes = i32, [vp, vp]
    L.qipb200_kernel_launches.restype, L.qipb200_kernel_launches.argtypes = u64, [vp]
    L.qipb200_kernel_counts.restype, L.qipb200_kernel_counts.argtypes = i32, [vp, vp, C.c_size_t]
    L.qipb200_release_pool.restype, L.qipb200_release_pool.argtypes = i32, [vp]
    L.qipb200_validate_op.restype, L.qipb200_validate_op.argtypes = i32, [vp, i32, u32, opp]
    for name in ("qipb200_apply_op", "qipb200_apply_op_overwrite"):
        f = getattr(L, name)
        f.restype, f.argtypes = i32, [vp, i32, u32, opp, vp, u64, vp, u64, u64, u64]
    L.qipb200_apply_ops.restype = i32
    L.qipb200_apply_ops.argtypes = [vp, i32, u32, opp, C.c_size_t, vp, u64, vp, u64, u64, u64]
    L.qipb200_state_new.restype, L.qipb200_state_new.argtypes = i32, [vp, i32, u32, C.POINTER(vp)]
    L.qipb200_state_free.restype, L.qipb200_state_free.argtypes = None, [vp]
    L.qipb200_state_set_basis.restype, L.qipb200_state_set_basis.argtypes = i32, [vp, u64]
    L.qipb200_state_upload.restype, L.qipb200_state_upload.argtypes = i32, [vp, vp, u64, u64]
    L.qipb200_state_download.restype, L.qipb200_state_download.argtypes = i32, [vp, vp, u64, u64]
    L.qipb200_state_apply_op.restype, L.qipb200_state_apply_op.argtypes = i32, [vp, opp]
    L.qipb200_state_apply_schedule.restype = i32
    L.qipb200_state_apply_schedule.argtypes = [vp, opp, C.c_size_t, u32]
    L.qipb200_state_norm2.restype, L.qipb200_state_norm2.argtypes = i32, [vp, C.POINTER(C.c_double)]
    L.qipb200_state_sync.restype, L.qipb200_state_sync.argtypes = i32, [vp]
    L.qipb200_state_max_abs_diff.restype = i32
    L.qipb200_state_max_abs_diff.argtypes = [vp, vp, C.POINTER(C.c_double)]
    L.qipb200_calculate_state.restype = i32
    L.qipb200_calculate_state.argtypes = [vp, i32, u32, u64, opp, C.c_size_t, u32, vp]
    L.qipb200_state_measure_probs.restype = i32
    L.qipb200_state_measure_probs.argtypes = [vp, vp, u32, vp]
    L.qipb200_state_measure_prob.restype = i32
    L.qipb200_state_measure_prob.argtypes = [vp, u64, vp, u32, C.POINTER(C.c_double)]
    L.qipb200_state_soft_measure.restype = i32
    L.qipb200_state_soft_measure.argtypes = [vp, vp, u32, C.c_double, C.POINTER(u64)]
    L.qipb200_state_sample.restype = i32
    L.qipb200_state_sample.argtypes = [vp, vp, u32, vp, u64, vp]
    L.qipb200_state_collapse.restype = i32
    L.qipb200_state_collapse.argtypes = [vp, vp, u32, u64, C.c_double]
    L.qipb200_state_measure.restype = i32
    L.qipb200_state_measure.argtypes = [vp, vp, u32, C.c_double, u32, C.POINTER(u64), C.POINTER(C.c_double)]
    L.qipb200_state_expect_paulis.restype = i32
    L.qipb200_state_expect_paulis.argtypes = [vp, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_expect_plan.restype = i32
    L.qipb200_expect_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, C.POINTER(u32)]
    L.qipb200_state_transition_paulis.restype = i32
    L.qipb200_state_transition_paulis.argtypes = [vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_transition_plan.restype = i32
    L.qipb200_transition_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_state_reduced_density.restype = i32
    L.qipb200_state_reduced_density.argtypes = [vp, vp, u32, vp]
    L.qipb200_state_purity.restype = i32
    L.qipb200_state_purity.argtypes = [vp, vp, u32, vp]
    L.qipb200_purity_plan.restype = i32
    L.qipb200_purity_plan.argtypes = [i32, u32, vp, u32, vp]
    L.qipb200_state_entanglement_spectrum.restype = i32
    L.qipb200_state_entanglement_spectrum.argtypes = [vp, vp, u32, vp, C.c_size_t, vp, vp]
    L.qipb200_entanglement_spectrum_plan.restype = i32
    L.qipb200_entanglement_spectrum_plan.argtypes = [i32, u32, vp, u32, vp]
    L.qipb200_state_apply_pauli_rotations.restype = i32
    L.qipb200_state_apply_pauli_rotations.argtypes = [vp, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_pauli_rotation_plan.restype = i32
    L.qipb200_pauli_rotation_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, C.POINTER(u32)]
    L.qipb200_state_apply_channels.restype = i32
    L.qipb200_state_apply_channels.argtypes = [vp, C.c_size_t, vp, vp, vp, vp, vp, C.POINTER(C.c_double)]
    L.qipb200_channels_plan.restype = i32
    L.qipb200_channels_plan.argtypes = [i32, u32, C.c_size_t, vp, vp, vp, vp]
    L.qipb200_state_apply_multiqubit_channels.restype = i32
    L.qipb200_state_apply_multiqubit_channels.argtypes = [vp, C.c_size_t, vp, vp, vp, vp, vp, vp,
                                                          C.POINTER(C.c_double)]
    L.qipb200_multiqubit_channels_plan.restype = i32
    L.qipb200_multiqubit_channels_plan.argtypes = [i32, u32, C.c_size_t, vp, vp, vp, vp, vp]
    L.qipb200_state_apply_kraus_channels.restype = i32
    L.qipb200_state_apply_kraus_channels.argtypes = [vp, C.c_size_t, vp, vp, vp, vp, vp, vp, vp,
                                                     C.POINTER(C.c_double)]
    L.qipb200_kraus_channels_plan.restype = i32
    L.qipb200_kraus_channels_plan.argtypes = [i32, u32, C.c_size_t, vp, vp, vp, vp, vp]
    sz = C.c_size_t
    L.qipb200_density_apply.restype = i32
    L.qipb200_density_apply.argtypes = [vp, opp, sz, sz, vp, vp, vp, vp, vp, u32]
    L.qipb200_density_schedule.restype = i32
    L.qipb200_density_schedule.argtypes = [i32, u32, opp, sz, sz, vp, vp, vp, vp, vp, vp, sz, C.POINTER(sz)]
    L.qipb200_density_from_state.restype, L.qipb200_density_from_state.argtypes = i32, [vp, vp]
    L.qipb200_density_measure_probs.restype = i32
    L.qipb200_density_measure_probs.argtypes = [vp, vp, u32, vp]
    L.qipb200_density_expect_paulis.restype = i32
    L.qipb200_density_expect_paulis.argtypes = [vp, vp, vp, vp, sz, vp]
    L.qipb200_density_reduced.restype, L.qipb200_density_reduced.argtypes = i32, [vp, vp, u32, vp]
    L.qipb200_density_fidelity.restype, L.qipb200_density_fidelity.argtypes = i32, [vp, vp, vp]
    L.qipb200_density_spectrum.restype, L.qipb200_density_spectrum.argtypes = i32, [vp, vp]
    L.qipb200_function_new.restype = i32
    L.qipb200_function_new.argtypes = [vp, u32, u32, vp, vp, C.POINTER(vp)]
    L.qipb200_function_free.restype, L.qipb200_function_free.argtypes = None, [vp]
    L.qipb200_state_apply_function.restype = i32
    L.qipb200_state_apply_function.argtypes = [vp, vp, vp, vp]
    L.qipb200_function_plan.restype = i32
    L.qipb200_function_plan.argtypes = [i32, u32, vp, u32, vp, u32, vp]
    L.qipb200_function_new_code.restype = i32
    L.qipb200_function_new_code.argtypes = [vp, u32, u32, C.c_char_p, u32, u32, C.c_char_p, C.c_size_t,
                                            C.POINTER(vp)]
    L.qipb200_function_set_params.restype = i32
    L.qipb200_function_set_params.argtypes = [vp, vp, u32]
    L.qipb200_function_code_compile.restype = i32
    L.qipb200_function_code_compile.argtypes = [u32, u32, C.c_char_p, u32, u32, C.c_char_p, C.c_size_t]
    L.qipb200_function_tabulate.restype = i32
    L.qipb200_function_tabulate.argtypes = [vp, u64, u64, vp, vp]
    L.qipb200_state_expect_function.restype = i32
    L.qipb200_state_expect_function.argtypes = [vp, vp, vp, vp]
    L.qipb200_state_apply_pauli_sum.restype = i32
    L.qipb200_state_apply_pauli_sum.argtypes = [vp, vp, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_pauli_sum_plan.restype = i32
    L.qipb200_pauli_sum_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, C.POINTER(u32)]
    L.qipb200_state_pauli_energy_gradient.restype = i32
    L.qipb200_state_pauli_energy_gradient.argtypes = [vp, vp, vp, vp, vp, C.c_size_t, vp, vp, vp, vp, C.c_size_t, vp,
                                                      vp, vp]
    L.qipb200_pauli_gradient_plan.restype = i32
    L.qipb200_pauli_gradient_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, vp, vp, vp, C.c_size_t,
                                              C.POINTER(u32)]
    L.qipb200_state_pauli_geometric_tensor.restype = i32
    L.qipb200_state_pauli_geometric_tensor.argtypes = [vp, vp, vp, vp, vp, vp, C.c_size_t, vp, vp, vp]
    L.qipb200_pauli_geometric_tensor_plan.restype = i32
    L.qipb200_pauli_geometric_tensor_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_state_evolve_pauli_sum.restype = i32
    L.qipb200_state_evolve_pauli_sum.argtypes = [vp, vp, vp, vp, vp, vp, C.c_size_t, vp, C.c_double, C.c_double,
                                                 C.POINTER(u32), C.POINTER(C.c_double)]
    L.qipb200_pauli_evolution_plan.restype = i32
    L.qipb200_pauli_evolution_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, vp, C.c_double, C.c_double, vp,
                                               C.POINTER(C.c_double), vp, C.c_size_t]
    L.qipb200_state_lanczos_pauli_sum.restype = i32
    L.qipb200_state_lanczos_pauli_sum.argtypes = [vp, vp, vp, vp, vp, vp, C.c_size_t, vp, u32, C.c_double, u32,
                                                  C.POINTER(u32), C.POINTER(u32), vp, vp, vp]
    L.qipb200_pauli_lanczos_plan.restype = i32
    L.qipb200_pauli_lanczos_plan.argtypes = [i32, u32, vp, vp, vp, C.c_size_t, vp]
    L.qipb200_lanczos_ritz.restype = i32
    L.qipb200_lanczos_ritz.argtypes = [vp, vp, u32, C.POINTER(C.c_double), vp, C.POINTER(C.c_double)]
    L.qipb200_state_new_sharded.restype = i32
    L.qipb200_state_new_sharded.argtypes = [vp, i32, u32, i32, i32, C.POINTER(vp)]
    L.qipb200_state_ipc_export.restype, L.qipb200_state_ipc_export.argtypes = i32, [vp, vp, vp]
    L.qipb200_state_ipc_import.restype, L.qipb200_state_ipc_import.argtypes = i32, [vp, vp, vp]
    L.qipb200_state_qubit_map.restype, L.qipb200_state_qubit_map.argtypes = i32, [vp, vp]
    L.qipb200_state_exchange_bytes.restype = i32
    L.qipb200_state_exchange_bytes.argtypes = [vp, C.POINTER(u64)]
    L.qipb200_plan_exchanges.restype = i32
    L.qipb200_plan_exchanges.argtypes = [i32, u32, i32, opp, C.c_size_t, vp]
    L.qipb200_state_save.restype, L.qipb200_state_save.argtypes = i32, [vp, C.c_char_p]
    L.qipb200_state_load.restype, L.qipb200_state_load.argtypes = i32, [vp, C.c_char_p]
    L.qipb200_schedule_parse.restype = i32
    L.qipb200_schedule_parse.argtypes = [vp, C.c_size_t, C.POINTER(vp), C.c_char_p, C.c_size_t]
    L.qipb200_schedule_ops.restype = opp
    L.qipb200_schedule_ops.argtypes = [vp, C.POINTER(C.c_size_t), C.POINTER(u32), C.POINTER(i32)]
    L.qipb200_schedule_free.restype, L.qipb200_schedule_free.argtypes = None, [vp]
    L.qipb200_schedule_serialise.restype = C.c_size_t
    L.qipb200_schedule_serialise.argtypes = [i32, u32, opp, C.c_size_t, vp, C.c_size_t]
    _lib = L
    return L


def check(status: int, ctx=None):
    """Non-zero status -> CircuitError(msg) (the shim's mapping, SURVEY.md section 8b)."""
    if status != 0:
        msg = lib().qipb200_last_error(ctx).decode("utf-8", "replace")
        raise CircuitError(msg or ("qipb200 status %d" % status), status=status)
