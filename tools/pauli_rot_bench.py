"""Time State.apply_pauli_rotations (qipb200_state_apply_pauli_rotations) on the N=30 f64 headline state, natively and
as apply_schedule (fused) of the CNOT-ladder decomposition, against the floor of one single-sweep fused pass (read and
write of the state) and one norm2 (read only).

    python tools/pauli_rot_bench.py OUTDIR [--n 30] [--repeats 5]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Workloads (angles seeded):
  (a) one transverse-field Ising Trotter step: n Z_iZ_i+1 (periodic), then n X_i;
  (b) a 3-regular QAOA layer: the ring and the diameters as 3n/2 Z_iZ_j cost terms, then n X_i mixers;
  (c) 64 UCC-style Jordan-Wigner strings (X/Y on 4 qubits, Z between them; seed 64);
  (d) the n + n(n-1)/2 diagonal terms Z_i and Z_iZ_j.
The floor is apply_schedule of one layer of rz on every qubit (one fused pass).  Each number is the median of the
repeats of a host clock around the call and a synchronise, after one warm-up.  Reported with the sweeps from
pauli_rotation_plan, the kernels launched, and ms / (sweeps * floor); the card's name and power limit are read in the
same run.  Writes OUTDIR/pauli_rot_bench.json."""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import pauli_rot_ref as rr  # noqa: E402
from rustqip_b200 import circuits, gates  # noqa: E402
from rustqip_b200.state import Context, State, pauli_rotation_plan  # noqa: E402


def gpu_info():
    q = "name,power.limit,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=" + q, "--format=csv,noheader"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
    except (OSError, subprocess.TimeoutExpired):
        out = ""
    f = [x.strip() for x in out.split(",")] if out else []
    return {"name": f[0] if f else None, "power_limit": f[1] if len(f) > 1 else None,
            "sm_max_clock": f[2] if len(f) > 2 else None}


def workloads(n):
    return {"a_ising_step": rr.ising_step(n), "b_qaoa_layer": rr.qaoa_layer(n), "c_ucc_64": rr.ucc_strings(n, 64, 64),
            "d_z_pairs": rr.z_pairs(n)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    rng = np.random.default_rng(30)
    wl = {k: (t, rng.uniform(-1, 1, size=len(t))) for k, t in workloads(n).items()}
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}}
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
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
                launches = ctx.kernel_launches() - l0
                times = []
                for _ in range(reps):
                    t0 = time.perf_counter()
                    fn()
                    st.sync()
                    times.append((time.perf_counter() - t0) * 1e3)
                return float(np.median(times)), times, launches

            rz_layer = [gates.rz(q, 0.1) for q in range(n)]
            floor, floor_all, floor_k = timed(lambda: st.apply_schedule(rz_layer))
            norm, norm_all, _ = timed(st.norm2)
            res["floor_fused_pass_ms"], res["floor_all_ms"], res["floor_kernels"] = floor, floor_all, floor_k
            res["norm2_ms"], res["norm2_all_ms"] = norm, norm_all
            for k, (terms, angles) in wl.items():
                sweeps = pauli_rotation_plan(n, np.complex128, terms)
                ops = rr.decompose_all(terms, angles)
                med, all_ms, launches = timed(lambda: st.apply_pauli_rotations(terms, angles))
                dmed, dall, dlaunches = timed(lambda: st.apply_schedule(ops))
                res["workloads"][k] = {
                    "terms": len(terms), "sweeps": sweeps, "kernels": launches, "ms": med, "all_ms": all_ms,
                    "x_sweeps_floor": med / (sweeps * floor),
                    "decomposition_ops": len(ops), "decomposition_kernels": dlaunches, "decomposition_ms": dmed,
                    "decomposition_all_ms": dall, "native_speedup": dmed / med}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "pauli_rot_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
