"""Time exact density-matrix simulation (DensityMatrix, qipb200_density_*) on a 15-qubit f64 rho (a 30-qubit vector,
16 GiB), against the same run's sweeps.

    python tools/density_bench.py OUTDIR [--n 15] [--repeats 5]

Rows:
  noisy     H layer, then 20 random {H, T, CNOT} layers (circuits.noisy_random_circuit, seed 0x5EED0015), each followed
            by amplitude damping (1e-3) and dephasing (1e-3) on every qubit, in one density_apply from a pending |0><0|:
            tile passes, total time, time per pass, and the same with fusion off.  Target: per pass <= 1.15 x a
            read-write sweep.
  noisy2q   the same with two-qubit depolarizing (1e-2) after each CNOT (4-qubit superoperators): the passes without a
            generated kernel (qipb200_jit_precompile) and the time, reported only.
  fidelity  <psi|rho|psi>, target <= 1.2 x a norm2 read sweep of the vector.
  set_pure  rho = |psi><psi|, target <= 1.0 x a read-write sweep.
  expect    the n + n (n - 1) / 2 Z_i and Z_i Z_j terms; reduced with k = 1, 6 and 10; measure_probs of all qubits; and
            spectrum at n = 13 against torch.linalg.eigvalsh of the downloaded matrix: reported only.
The sweeps: norm2 of the vector (a read sweep) and one unfused single-qubit gate on it (a read-write sweep).  Each
number is the median of the repeats of a host clock around a call that ends in a device synchronise, after one
warm-up; the card's name and power limit are read in the same run.  Writes OUTDIR/density_bench.json."""
import argparse
import ctypes as C
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from channel_bench import gpu_info  # noqa: E402
from rustqip_b200 import _lib, circuits, gates  # noqa: E402
from rustqip_b200._abi import marshal_ops, prec_of  # noqa: E402
from rustqip_b200.state import Context, DensityMatrix, State, density_schedule  # noqa: E402


def timed(fn, reps, sync):
    fn()
    sync()
    ts = []
    for _ in range(reps):
        t0 = time.perf_counter()
        fn()
        sync()
        ts.append((time.perf_counter() - t0) * 1e3)
    return statistics.median(ts), ts


def unjitted_passes(n, items):
    ops = density_schedule(n, np.complex128, items)
    arr, keep = marshal_ops(ops, prec_of(np.complex128))
    out = (C.c_double * 5)()
    log = C.create_string_buffer(4000)
    rc = _lib.lib().qipb200_jit_precompile(prec_of(np.complex128), 2 * n, arr, len(ops), out, log, 4000)
    return {"rc": rc, "passes": int(out[0]), "generated": int(out[1]), "compiled": int(out[2]),
            "without_generated_kernel": int(out[0] - out[1]), "ops": len(ops)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=15)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(3, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    res = {"gpu": gpu_info(), "n": n, "vector_qubits": 2 * n, "dtype": "complex128", "repeats": reps}
    noisy = circuits.noisy_random_circuit(n, 20, 0x5EED0015)
    noisy2 = circuits.noisy_random_circuit(n, 20, 0x5EED0015, cnot_depolarizing=1e-2)
    with Context(0) as ctx:
        with DensityMatrix(n, np.complex128, ctx) as rho, State(n, np.complex128, ctx) as psi:
            sync = rho.state.sync
            psi.upload(circuits.random_state(n, 15, np.complex128))
            rho.set_pure(psi)
            res["read_sweep_ms"], _ = timed(lambda: rho.state.norm2(), reps, sync)
            res["rw_sweep_ms"], _ = timed(lambda: rho.state.apply_schedule([gates.h(0)], fusion=False), reps, sync)
            rw, rd = res["rw_sweep_ms"], res["read_sweep_ms"]

            def run(items, fusion=True):
                rho.set_basis(0)
                rho.apply(items, fusion=fusion)

            for name, items in (("noisy", noisy), ("noisy2q", noisy2)):
                before = ctx.launch_stats()["tile_passes"]
                run(items)
                sync()
                passes = ctx.launch_stats()["tile_passes"] - before
                ms, ts = timed(lambda: run(items), reps, sync)
                res[name] = {"ms": ms, "samples_ms": ts, "tile_passes": passes,
                             "ms_per_pass": ms / max(1, passes), "per_pass_over_rw_sweep": ms / max(1, passes) / rw,
                             "jit": ctx.jit_stats(wait=True)["note"]}
            res["noisy2q"]["precompile"] = unjitted_passes(n, noisy2)
            res["noisy"]["precompile"] = unjitted_passes(n, noisy)
            t0 = time.perf_counter()
            run(noisy, fusion=False)
            sync()
            res["noisy"]["fusion_off_ms"] = (time.perf_counter() - t0) * 1e3
            rho.set_pure(psi)
            ms, _ = timed(lambda: rho.fidelity(psi), reps, sync)
            res["fidelity"] = {"ms": ms, "over_read_sweep": ms / rd}
            ms, _ = timed(lambda: rho.set_pure(psi), reps, sync)
            res["set_pure"] = {"ms": ms, "over_rw_sweep": ms / rw}
            run(noisy)
            terms = [[("Z", i)] for i in range(n)] + [[("Z", i), ("Z", j)] for i in range(n) for j in range(i + 1, n)]
            ms, _ = timed(lambda: rho.expect_paulis(terms), reps, sync)
            res["expect"] = {"terms": len(terms), "ms": ms}
            for k in (1, 6, 10):
                ms, _ = timed(lambda: rho.reduced_density(list(range(k))), reps, sync)
                res["reduced_k%d" % k] = {"ms": ms}
            ms, _ = timed(lambda: rho.measure_probs(list(range(n))), reps, sync)
            res["measure_probs_all"] = {"ms": ms}
        m = 13
        with DensityMatrix(m, np.complex128, ctx) as rho:
            rho.set_basis(0)
            rho.apply(circuits.noisy_random_circuit(m, 4, 0x5EED0013, gamma=0.05, lam=0.05))
            ms, _ = timed(lambda: rho.spectrum(), 3, rho.state.sync)
            ours = rho.spectrum()
            res["spectrum_n13"] = {"ms": ms}
            try:
                import torch
                a = torch.from_numpy(rho.download()).cuda()
                ms2, _ = timed(lambda: torch.linalg.eigvalsh(a), 3, torch.cuda.synchronize)
                ev = torch.linalg.eigvalsh(a).cpu().numpy()[::-1]
                res["spectrum_n13"].update({"torch_eigvalsh_ms": ms2, "max_abs_diff": float(np.max(np.abs(ev - ours)))})
            except Exception as e:  # torch without CUDA: report, do not fall back
                res["spectrum_n13"]["torch_error"] = repr(e)
    path = os.path.join(args.outdir, "density_bench.json")
    with open(path, "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items()}, default=str)[:4000])


if __name__ == "__main__":
    main()
