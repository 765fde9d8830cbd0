"""Time State.lanczos_pauli_sum (qipb200_state_lanczos_pauli_sum) on N=30 f64 states against apply_pauli_sum on the
same terms and against the read-sweep floor (norm2).

    python tools/lanczos_bench.py OUTDIR [--n 30] [--max-steps 300]

Three f64 states of 2^N amplitudes are needed (48 GiB at N=30); when the card cannot hold them the run falls back to
N-1 and records it.  Start state: R_Y(0.3) on every qubit, then a random {H,T,CNOT} circuit of depth 4 (seed
0x5EED0003): spread out, with weight on every symmetry sector.  Workloads (seeded):
  (a) the open transverse-field Ising chain, J_i ~ U(0.2, 0.6), h_i ~ U(0.9, 1.3) (paramagnetic), with the energy
      error against the free-fermion closed form;
  (b) the open Heisenberg XXX chain, 0.25 (X_iX_i+1 + Y_iY_i+1 + Z_iZ_i+1);
  (c) the 64 UCC-style strings of tools/pauli_rot_bench.py (seed 64) with 0.1 x N(0, 1) coefficients.
Each call is timed once with a host clock around the call (which synchronises), after a two-step warm-up; each
workload runs energy only, then vector mode from the same start state.  Reported: steps, converged, energy, residual,
call ms in both modes, ms per first-pass step (energy-only call / steps), ms per second-pass step ((vector call -
energy-only call - tail) / (steps - 1), the tail priced at apply_pauli_sum + 3 norm2), apply_pauli_sum ms (median of
3) and norm2 ms.  Targets, each state transfer beyond apply_pauli_sum priced at one norm2: a first-pass step <=
apply_pauli_sum + 1.25 x 4 norm2 (the read of u_(j-1), the update sweep's two reads and one write), a second-pass step
<= apply_pauli_sum + 1.25 x 6 norm2 (plus the read and write of the state).  The card's name and power limit are read
in the same run.  Writes OUTDIR/lanczos_bench.json."""
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

import lanczos_ref as lr  # noqa: E402
import pauli_rot_ref as rr  # noqa: E402
from pauli_rot_bench import gpu_info  # noqa: E402
from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.errors import CircuitError  # noqa: E402
from rustqip_b200.state import Context, State, pauli_lanczos_plan  # noqa: E402

FIRST_EXTRA, SECOND_EXTRA = 4, 6


def workloads(n):
    rng = np.random.default_rng(30)
    J, h = rng.uniform(0.2, 0.6, size=n - 1), rng.uniform(0.9, 1.3, size=n)
    ucc = rr.ucc_strings(n, 64, 64)
    return {"a_tfim": (lr.tfim(J, h), lr.tfim_ground(J, h)), "b_xxx": (lr.heisenberg(n), None),
            "c_ucc_64": ((ucc, 0.1 * np.random.default_rng(3).normal(size=len(ucc))), None)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--max-steps", type=int, default=300)
    a = ap.parse_args()
    os.makedirs(a.outdir, exist_ok=True)
    res = {"gpu": gpu_info(), "dtype": "f64", "max_steps": a.max_steps, "tol": 1e-8, "workloads": {}}
    with Context(0) as ctx:
        n = a.n
        states = []
        while not states:
            try:
                states = [State(n, np.complex128, ctx) for _ in range(3)]
            except CircuitError as e:
                for s in states:
                    s.free()
                states = []
                res.setdefault("fallback", []).append("n=%d: %s" % (n, str(e)[:200]))
                ctx.release_pool()
                n -= 1
        res["n"] = n
        st, wa, wb = states

        def prepare():
            st.set_basis(0)
            st.apply_pauli_rotations([[("Y", q)] for q in range(n)], np.full(n, 0.3))
            st.apply_schedule(circuits.random_circuit(n, 4, 0x5EED0003, "H,T,CNOT"))
            st.sync()

        def clock(fn):
            st.sync()
            t0 = time.perf_counter()
            out = fn()
            st.sync()
            return (time.perf_counter() - t0) * 1e3, out

        prepare()
        norm_ms = float(np.median([clock(st.norm2)[0] for _ in range(5)]))
        res["norm2_ms"] = norm_ms
        for name, ((terms, coeffs), exact) in workloads(n).items():
            plan = pauli_lanczos_plan(n, np.complex128, terms)
            sum_ms = float(np.median([clock(lambda: wa.apply_pauli_sum(st, terms, coeffs))[0] for _ in range(3)]))
            st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=2, vector=False)  # warm-up
            e_ms, r0 = clock(lambda: st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=a.max_steps, vector=False))
            l0 = ctx.kernel_launches()
            v_ms, r = clock(lambda: st.lanczos_pauli_sum(wa, wb, terms, coeffs, max_steps=a.max_steps))
            launched = ctx.kernel_launches() - l0
            m = r.steps
            first = e_ms / max(1, m)
            second = (v_ms - e_ms - (sum_ms + 3 * norm_ms)) / max(1, m - 1)
            w = {"terms": len(terms), "plan": plan, "launched_vector": launched, "steps": m,
                 "converged": r.converged, "energy_only": r0.energy, "estimate": r0.residual, "energy": r.energy,
                 "residual": r.residual, "ritz_norm": r.ritz_norm, "call_ms_energy_only": e_ms,
                 "call_ms_vector": v_ms, "ms_per_first_pass_step": first, "ms_per_second_pass_step": second,
                 "apply_pauli_sum_ms": sum_ms,
                 "target_first_ms": sum_ms + 1.25 * FIRST_EXTRA * norm_ms,
                 "target_second_ms": sum_ms + 1.25 * SECOND_EXTRA * norm_ms}
            w["target_first_met"] = first <= w["target_first_ms"]
            w["target_second_met"] = second <= w["target_second_ms"]
            if exact is not None:
                w["closed_form"] = exact
                w["energy_error"] = r.energy - exact
            res["workloads"][name] = w
            print(name, json.dumps(w), flush=True)
            prepare()
        for s in states:
            s.free()
    with open(os.path.join(a.outdir, "lanczos_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "workloads"}))


if __name__ == "__main__":
    main()
