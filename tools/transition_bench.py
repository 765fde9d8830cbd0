"""Time State.transition_paulis / State.overlap (qipb200_state_transition_paulis) on two N=30 f64 states against the
one-state calls they generalise, and the host alternative (downloading both states).

    python tools/transition_bench.py OUTDIR [--n 30] [--repeats 5] [--corr-n 28] [--corr-points 3]

States: the headline random {H,T,CNOT} circuit, depth 40, from |0>, with seed 0x5EED0002 (ket) and 0x5EED0003 (bra).
Workloads (targets in brackets):
  (a) overlap alone                                   [<= 1.25 x (2 x norm2)]
  (b) the n + n(n-1)/2 terms Z_i and Z_iZ_j            [<= 2 x expect_paulis of the same terms on one state]
  (c) the TFIM: n X_i and n Z_iZ_{i+1} (periodic)       [<= 2 x expect_paulis of the same terms on one state]
  (d) downloading both states into pinned host memory (the host alternative)
  (e) a correlation run at N=corr-n f64 in four states: phi = Z_0 psi (apply_pauli_sum), then per time point psi and
      phi each evolve by dt = 0.1 under the TFIM (evolve_pauli_sum, sharing the two work states) and one call gives
      every <psi(t)|Z_i|phi(t)>; the time per time point
  (f) tile-pair sweeps: X^n, X_0 X_(n-1) and Y_0 Z_1 X_(n-1), against expect_paulis of the same terms
Each one-call workload is the median of the repeats of a host clock around a synchronising call, after one warm-up.
The card's name and power limit are read in the same run.  Writes OUTDIR/transition_bench.json."""
import argparse
import itertools
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from expect_bench import gpu_info  # noqa: E402
from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.state import Context, State, expect_plan, transition_plan  # noqa: E402


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def tfim(n):
    return [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]


def measure(ctx, fn, reps):
    fn()  # warm-up
    l0 = ctx.kernel_launches()
    fn()
    launches = ctx.kernel_launches() - l0
    times = [clock(fn) for _ in range(reps)]
    return {"median_ms": float(np.median(times)), "all_ms": times, "kernel_launches": launches}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--corr-n", type=int, default=28)
    ap.add_argument("--corr-points", type=int, default=3)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    import torch
    diag = [[("Z", i)] for i in range(n)] + [[("Z", i), ("Z", j)] for i, j in itertools.combinations(range(n), 2)]
    pair = [[("X", q) for q in range(n)], [("X", 0), ("X", n - 1)], [("Y", 0), ("Z", 1), ("X", n - 1)]]
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "states": "random {H,T,CNOT} depth 40 from |0>, seeds 0x5EED0002 (ket) and 0x5EED0003 (bra)",
           "workloads": {}}
    w = res["workloads"]
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as ket, State(n, np.complex128, ctx) as bra:
            for st, seed in ((ket, 0x5EED0002), (bra, 0x5EED0003)):
                st.set_basis(0)
                st.apply_schedule(circuits.random_circuit(n, 40, seed, "H,T,CNOT"))
            ket.sync()
            w["norm2"] = measure(ctx, ket.norm2, reps)
            w["a_overlap"] = measure(ctx, lambda: bra.overlap(ket), reps)
            w["a_overlap"]["plan"] = transition_plan(n, np.complex128, [[]])
            for key, terms in (("b_diagonal", diag), ("c_ising", tfim(n)), ("f_tile_pairs", pair)):
                w[key] = measure(ctx, lambda t=terms: bra.transition_paulis(ket, t), reps)
                w[key]["terms"] = len(terms)
                w[key]["plan"] = transition_plan(n, np.complex128, terms)
                w[key + "_expect"] = measure(ctx, lambda t=terms: ket.expect_paulis(t), reps)
                w[key + "_expect"]["sweeps"] = expect_plan(n, np.complex128, terms)
            host = torch.empty(16 << n, dtype=torch.uint8, pin_memory=True)

            def download_both():
                ket.download_ptr(host.data_ptr(), 1 << n)
                bra.download_ptr(host.data_ptr(), 1 << n)

            w["d_download_both"] = measure(ctx, download_both, reps)
            del host
        ctx.release_pool()
        m = args.corr_n
        h = tfim(m)
        coeffs = [1.0] * m + [1.0] * m
        zs = [[("Z", i)] for i in range(m)]
        with State(m, np.complex128, ctx) as psi, State(m, np.complex128, ctx) as phi, \
                State(m, np.complex128, ctx) as wa, State(m, np.complex128, ctx) as wb:
            psi.set_basis(0)
            psi.apply_schedule(circuits.random_circuit(m, 40, 0x5EED0002, "H,T,CNOT"))
            phi.apply_pauli_sum(psi, [[("Z", 0)]], [1.0])

            def point():
                k1 = psi.evolve_pauli_sum(wa, wb, h, coeffs, 0.1)[0]
                k2 = phi.evolve_pauli_sum(wa, wb, h, coeffs, 0.1)[0]
                phi.sync()  # the evolutions are stream-ordered: time the transition call alone
                t0 = time.perf_counter()
                c = psi.transition_paulis(phi, zs)
                return k1 + k2, (time.perf_counter() - t0) * 1e3, c

            point()  # warm-up
            times, corr_ms = [], []
            for _ in range(args.corr_points):
                t0 = time.perf_counter()
                deg, cms, c = point()
                times.append((time.perf_counter() - t0) * 1e3)
                corr_ms.append(cms)
            w["e_correlation_point"] = {"n": m, "median_ms": float(np.median(times)), "all_ms": times,
                                        "transition_ms": corr_ms, "chebyshev_degrees_per_point": deg,
                                        "last_C_0j": [float(v.real) for v in c[:4]]}
    nm = w["norm2"]["median_ms"]
    res["a_over_2x_norm2"] = w["a_overlap"]["median_ms"] / (2 * nm)
    res["b_over_expect"] = w["b_diagonal"]["median_ms"] / w["b_diagonal_expect"]["median_ms"]
    res["c_over_expect"] = w["c_ising"]["median_ms"] / w["c_ising_expect"]["median_ms"]
    res["f_over_expect"] = w["f_tile_pairs"]["median_ms"] / w["f_tile_pairs_expect"]["median_ms"]
    res["targets_met"] = {"a": res["a_over_2x_norm2"] <= 1.25, "b": res["b_over_expect"] <= 2.0,
                          "c": res["c_over_expect"] <= 2.0}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "transition_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
