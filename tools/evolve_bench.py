"""Time State.evolve_pauli_sum (qipb200_state_evolve_pauli_sum) on the N=30 f64 headline state against apply_pauli_sum on
the same terms and against the read-sweep floor (norm2).

    python tools/evolve_bench.py OUTDIR [--n 30] [--repeats 5]

Three f64 states of 2^N amplitudes are needed (48 GiB at N=30); when the card cannot hold them the run falls back to
N-1 and records it.  State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Workloads, t = 1, coefficients
0.1 x N(0, 1) seeded per workload (so that b = sum |c_h| and the degree stay moderate):
  (a) the 45-term 3-regular QAOA cost (1 sweep per step);
  (b) the transverse-field Ising model, n Z_iZ_i+1 and n X_i (4 sweeps per step at N=30);
  (c) the 64 UCC-style strings of tools/pauli_rot_bench.py (seed 64).
Each time is the median of the repeats of a host clock around the call and a synchronise, after a warm-up.  Reported
per workload: K, sweeps per step s, kernels, call ms, ms per step (call / K), apply_pauli_sum ms on the same terms (s
sweeps), and |norm2 after - norm2 before| over the repeats; norm2 ms is the read-sweep floor.  The target: a step costs
no more than apply_pauli_sum plus 1.25 x its 3 extra state transfers (the first sweep reads T_(k-1), the last reads
and writes the state), each priced at one norm2.  The card's name and power limit are read in the same run.
Writes OUTDIR/evolve_bench.json."""
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
from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.errors import CircuitError  # noqa: E402
from rustqip_b200.state import Context, State, pauli_evolution_plan  # noqa: E402

EXTRA_TRANSFERS = 3


def workloads(n):
    w = {"a_qaoa_cost": rr.qaoa_layer(n)[:45] if n == 30 else rr.qaoa_layer(n)[: n + n // 2],
         "b_tfim": rr.ising_step(n), "c_ucc_64": rr.ucc_strings(n, 64, 64)}
    return {k: (v, 0.1 * np.random.default_rng(i + 1).normal(size=len(v))) for i, (k, v) in enumerate(w.items())}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    a = ap.parse_args()
    os.makedirs(a.outdir, exist_ok=True)
    res = {"gpu": gpu_info(), "dtype": "f64", "t": 1.0, "repeats": a.repeats, "workloads": {}}
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
        st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
        st.sync()

        def timed(fn):
            fn()  # warm-up
            st.sync()
            ts = []
            for _ in range(a.repeats):
                t0 = time.perf_counter()
                fn()
                st.sync()
                ts.append((time.perf_counter() - t0) * 1e3)
            return float(np.median(ts)), ts

        norm_ms, _ = timed(st.norm2)
        res["norm2_ms"] = norm_ms
        for name, (terms, coeffs) in workloads(n).items():
            K, s, kernels, tail, _ = pauli_evolution_plan(n, np.complex128, terms, coeffs, 1.0, 1e-12)
            n0 = st.norm2()
            drift = []

            def evolve():
                st.evolve_pauli_sum(wa, wb, terms, coeffs, 1.0)

            l0 = ctx.kernel_launches()
            call_ms, ts = timed(evolve)
            launched = (ctx.kernel_launches() - l0) // (a.repeats + 1)
            drift.append(abs(st.norm2() - n0))
            sum_ms, _ = timed(lambda: wa.apply_pauli_sum(st, terms, coeffs))
            step_ms = call_ms / K
            limit = sum_ms + 1.25 * EXTRA_TRANSFERS * norm_ms
            res["workloads"][name] = {
                "terms": len(terms), "degree": K, "sweeps_per_step": s, "kernels": kernels, "launched": launched,
                "tail": tail, "call_ms": call_ms, "call_ms_all": ts, "ms_per_step": step_ms,
                "apply_pauli_sum_ms": sum_ms, "step_minus_sum_ms": step_ms - sum_ms,
                "target_step_ms": limit, "target_met": step_ms <= limit,
                "norm2_drift_after_%d_calls" % (a.repeats + 1): max(drift)}
            print(name, json.dumps(res["workloads"][name]), flush=True)
        for s in states:
            s.free()
    with open(os.path.join(a.outdir, "evolve_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: v for k, v in res.items() if k != "workloads"}))


if __name__ == "__main__":
    main()
