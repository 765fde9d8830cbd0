"""Time State.expect_paulis (qipb200_state_expect_paulis) on the N=30 f64 headline state against one norm2 (the
single-read-sweep floor) and one download to pinned host memory (what evaluating observables on the host starts with).

    python tools/expect_bench.py OUTDIR [--n 30] [--repeats 5]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Workloads:
  (a) the n + n(n-1)/2 diagonal terms Z_i and Z_iZ_j;
  (b) the transverse-field Ising Hamiltonian: n X_i and n Z_iZ_{i+1} (periodic);
  (c) 2^10 random weight-4 strings (seed 1024);
  (d) one norm2;
  (e) one download of the whole state into pinned host memory.
Each is the median of the repeats of a host clock around a synchronising call, after one warm-up.  Reported with the
read sweeps from expect_plan, the algorithmic bytes (sweeps * 2^n * 16 B) and their fraction of 3.35 TB/s; the card's
name and power limit are read in the same run.  Writes OUTDIR/expect_bench.json."""
import argparse
import itertools
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.state import Context, State, expect_plan  # noqa: E402

PEAK_TBS = 3.35


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


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def workloads(n):
    diag = [[("Z", i)] for i in range(n)] + [[("Z", i), ("Z", j)] for i, j in itertools.combinations(range(n), 2)]
    tfim = [[("X", i)] for i in range(n)] + [[("Z", i), ("Z", (i + 1) % n)] for i in range(n)]
    rng = np.random.default_rng(1024)
    rand4 = [[(str(rng.choice(list("XYZ"))), int(q)) for q in rng.choice(n, size=4, replace=False)]
             for _ in range(1 << 10)]
    return {"a_diagonal": diag, "b_ising": tfim, "c_random_w4": rand4}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    import torch
    wl = workloads(n)
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}}
    amp_bytes = 16 << n
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()
            host = torch.empty(amp_bytes, dtype=torch.uint8, pin_memory=True)
            fns = {k: (lambda t=t: st.expect_paulis(t)) for k, t in wl.items()}
            fns["d_norm2"] = st.norm2
            fns["e_download_pinned"] = lambda: st.download_ptr(host.data_ptr(), 1 << n)
            for k, fn in fns.items():
                fn()  # warm-up
                l0 = ctx.kernel_launches()
                fn()
                launches = ctx.kernel_launches() - l0
                times = [clock(fn) for _ in range(reps)]
                sweeps = expect_plan(n, np.complex128, wl[k]) if k in wl else 1
                med = float(np.median(times))
                res["workloads"][k] = {
                    "terms": len(wl[k]) if k in wl else None, "sweeps": sweeps, "kernel_launches": launches,
                    "median_ms": med, "all_ms": times, "algorithmic_bytes": sweeps * amp_bytes,
                    "fraction_of_3.35TBs": sweeps * amp_bytes / (med * 1e-3) / (PEAK_TBS * 1e12)}
    w = res["workloads"]
    d = w["d_norm2"]["median_ms"]
    res["a_over_norm2"] = w["a_diagonal"]["median_ms"] / d
    res["b_over_sweeps_x_norm2"] = w["b_ising"]["median_ms"] / (w["b_ising"]["sweeps"] * d)
    res["c_over_sweeps_x_norm2"] = w["c_random_w4"]["median_ms"] / (w["c_random_w4"]["sweeps"] * d)
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "expect_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
