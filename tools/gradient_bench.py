"""Time State.energy_gradient (qipb200_state_pauli_energy_gradient) and State.apply_pauli_sum on the N=30 f64 headline
state, against the floor of one single-sweep fused pass and against the parameter-shift route through existing calls.

    python tools/gradient_bench.py OUTDIR [--n 30] [--repeats 5]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>; the work state is a second state of the same size.
Workloads (angles and coefficients seeded):
  (a) a 3-regular QAOA layer as the ansatz, its 3n/2 Z_iZ_j cost terms as H;
  (b) two transverse-field Ising Trotter steps as the ansatz, the TFIM (n Z_iZ_i+1, n X_i) as H;
  (c) 64 UCC-style Jordan-Wigner strings (seed 64) as the ansatz, the TFIM as H.
The floor is apply_schedule of one layer of rz on every qubit (one fused pass: one read and one write of the state).
Each number is the median of the repeats of a host clock around the call and a synchronise, after a warm-up and after
the generated kernels have compiled.  Reported per workload: the {forward, sum, backward} sweeps of pauli_gradient_plan
and the kernels launched; the ms of the whole call, of apply_pauli_sum alone and of apply_pauli_rotations alone; the
backward ms (whole call minus those two, so an estimate by difference) per backward sweep over twice the floor (a
backward sweep reads and writes two states); and one parameter-shift evaluation (the shifted rotations, expect_paulis of
H, the rotations undone) times 2T, labelled as that product.  The card's name and power limit are read in the same run.
Writes OUTDIR/gradient_bench.json."""
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
from rustqip_b200.state import Context, State, pauli_gradient_plan  # noqa: E402


def workloads(n):
    cost = rr.qaoa_layer(n)[: n + n // 2]
    tfim = rr.ising_step(n)
    return {"a_qaoa_layer": (rr.qaoa_layer(n), cost), "b_ising_2_steps": (rr.ising_step(n) * 2, tfim),
            "c_ucc_64": (rr.ucc_strings(n, 64, 64), tfim)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    rng = np.random.default_rng(31)
    wl = {k: (a, rng.uniform(-1, 1, size=len(a)), h, rng.normal(size=len(h))) for k, (a, h) in workloads(n).items()}
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}}
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st, State(n, np.complex128, ctx) as wk:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()

            def timed(fn):
                fn()  # warm-up
                ctx.jit_stats(wait=True)  # fused passes run on their generated kernels from here on
                fn()
                st.sync()
                l0 = ctx.kernel_launches()
                fn()
                st.sync()
                wk.sync()
                launches = ctx.kernel_launches() - l0
                times = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    fn()
                    st.sync()
                    times.append((time.perf_counter() - t0) * 1e3)
                return float(np.median(times)), times, launches

            rz_layer = [gates.rz(q, 0.1) for q in range(n)]
            floor, floor_all, _ = timed(lambda: st.apply_schedule(rz_layer))
            res["floor_fused_pass_ms"], res["floor_all_ms"] = floor, floor_all
            for k, (ansatz, angles, ham, coeffs) in wl.items():
                f, s, b = pauli_gradient_plan(n, np.complex128, ansatz, ham)
                T = len(ansatz)
                med, all_ms, launches = timed(lambda: st.energy_gradient(wk, ansatz, angles, ham, coeffs))
                smed, sall, _ = timed(lambda: wk.apply_pauli_sum(st, ham, coeffs))
                fmed, fall, _ = timed(lambda: st.apply_pauli_rotations(ansatz, angles))
                inv_terms, inv_angles = ansatz[::-1], -np.asarray(angles)[::-1]

                def shift_eval():
                    st.apply_pauli_rotations(ansatz, angles)
                    st.expect_paulis(ham)
                    st.apply_pauli_rotations(inv_terms, inv_angles)

                pmed, pall, _ = timed(shift_eval)
                back = med - smed - fmed
                res["workloads"][k] = {
                    "terms": T, "ham_terms": len(ham), "sweeps_forward_sum_backward": [f, s, b],
                    "kernels": launches, "ms": med, "all_ms": all_ms, "apply_pauli_sum_ms": smed,
                    "apply_pauli_sum_all_ms": sall, "forward_rotations_ms": fmed,
                    "backward_ms_by_difference": back, "backward_per_sweep_x_2floor": back / (b * 2 * floor),
                    "one_shift_evaluation_ms": pmed, "one_shift_evaluation_all_ms": pall,
                    "shift_evaluation_ms_times_2T": 2 * T * pmed, "speedup_vs_shift_estimate": 2 * T * pmed / med}
                print(k, json.dumps(res["workloads"][k]), flush=True)
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "gradient_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
