"""Time State.geometric_tensor (qipb200_state_pauli_geometric_tensor) on the N=30 f64 headline state, against the
floor of one single-sweep fused pass and against the same tensor computed through existing calls.

    python tools/qgt_bench.py OUTDIR [--n 30] [--repeats 3] [--route-forks K]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>; work_a and work_b are two more states of the same size
(48 GiB in all at N=30 f64).  Workloads (angles seeded):
  (a) a 3-regular QAOA layer (T = 75 at n = 30);
  (b) one transverse-field Ising Trotter step (T = 60);
  (c) 64 UCC-style Jordan-Wigner strings, seed 64 (T = 64).
The floor is apply_schedule of one layer of rz on every qubit (one fused pass: one read and one write of the state).
Each call is timed as the median of the repeats of a host clock around the call and a synchronise, after a warm-up
and after the generated kernels have compiled.  Each call moves the state on to U psi (the time does not depend on
the amplitudes).  Reported per workload: the plan counts
(forks, segment sweeps, kernels) and the kernels launched; the call's ms; call / ((forks + segment sweeps) x 2 x
floor), since a fork and a segment sweep each move four state passes; and the tensor through existing calls, run once:
per fork apply_pauli_rotations of R_i, apply_pauli_sum of the empty string (the copy) and of P_i, then per later term
transition_paulis of P_j between the work states and apply_pauli_rotations of R_j on both (with --route-forks K only
the first K forks run and the time is scaled by the share of steps they hold, labelled as an estimate).  Single-term
calls time the fork alone (one fork and the final reduction) on a low-bit X, a high-bit X and a Z string.  The card's
name and power limit are read in the same run.  Writes OUTDIR/qgt_bench.json."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests"), os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

import pauli_rot_ref as rr  # noqa: E402
from pauli_rot_bench import gpu_info  # noqa: E402
from rustqip_b200 import circuits, gates  # noqa: E402
from rustqip_b200.state import Context, State, pauli_geometric_tensor_plan  # noqa: E402


def workloads(n):
    return {"a_qaoa_layer": rr.qaoa_layer(n), "b_ising_step": rr.ising_step(n), "c_ucc_64": rr.ucc_strings(n, 64, 64)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    ap.add_argument("--route-forks", type=int, default=0, help="forks of the existing-call route to run (0: all)")
    args = ap.parse_args()
    n, reps = args.n, max(1, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    rng = np.random.default_rng(37)
    wl = {k: (a, rng.uniform(-1, 1, size=len(a))) for k, a in workloads(n).items()}
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}, "fork_alone": {}}
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st, State(n, np.complex128, ctx) as wa, \
                State(n, np.complex128, ctx) as wb:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()

            def timed(fn):
                fn()  # warm-up
                ctx.jit_stats(wait=True)  # fused passes run on their generated kernels from here on
                times, launches = [], None
                for _ in range(reps):
                    l0 = ctx.kernel_launches()
                    t0 = time.perf_counter()
                    fn()
                    st.sync()
                    times.append((time.perf_counter() - t0) * 1e3)
                    launches = ctx.kernel_launches() - l0
                return float(np.median(times)), times, launches

            rz_layer = [gates.rz(q, 0.1) for q in range(n)]
            floor, floor_all, _ = timed(lambda: st.apply_schedule(rz_layer))
            res["floor_fused_pass_ms"], res["floor_all_ms"] = floor, floor_all
            print("floor", floor, flush=True)
            for label, term in (("x_low_bit", [("X", n - 1)]), ("x_high_bit", [("X", 0)]),
                                ("z_string", [("Z", q) for q in range(0, n, 3)])):
                med, all_ms, launches = timed(lambda: st.geometric_tensor(wa, wb, [term], [0.3]))
                res["fork_alone"][label] = {"ms": med, "all_ms": all_ms, "kernels": launches,
                                            "x_2floor": med / (2 * floor)}
                print("fork", label, json.dumps(res["fork_alone"][label]), flush=True)
            for k, (ansatz, angles) in wl.items():
                T = len(ansatz)
                forks, sweeps, kernels = pauli_geometric_tensor_plan(n, np.complex128, ansatz)
                med, all_ms, launches = timed(lambda: st.geometric_tensor(wa, wb, ansatz, angles))

                K = T if args.route_forks <= 0 else min(T, args.route_forks)

                def route():
                    for i in range(K):
                        st.apply_pauli_rotations([ansatz[i]], [angles[i]])
                        wa.apply_pauli_sum(st, [[]], [1.0])
                        wb.apply_pauli_sum(st, [ansatz[i]], [1.0])
                        for j in range(i + 1, T):
                            wb.transition_paulis(wa, [ansatz[j]])
                            wa.apply_pauli_rotations([ansatz[j]], [angles[j]])
                            wb.apply_pauli_rotations([ansatz[j]], [angles[j]])

                t0 = time.perf_counter()
                route()
                st.sync()
                route_ms = (time.perf_counter() - t0) * 1e3
                steps_all = sum(1 + (T - 1 - i) for i in range(T))
                steps_run = sum(1 + (T - 1 - i) for i in range(K))
                route_est = route_ms * steps_all / steps_run
                res["workloads"][k] = {
                    "terms": T, "plan_forks_sweeps_kernels": [forks, sweeps, kernels], "kernels": launches,
                    "ms": med, "all_ms": all_ms, "x_forks_plus_sweeps_2floor": med / ((forks + sweeps) * 2 * floor),
                    "existing_calls_forks_run": K, "existing_calls_ms_run": route_ms,
                    "existing_calls_ms" + ("" if K == T else "_estimate"): route_est,
                    "speedup_vs_existing_calls": route_est / med}
                print(k, json.dumps(res["workloads"][k]), flush=True)
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "qgt_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
