"""Time State.reduced_density (qipb200_state_reduced_density) on the N=30 f64 headline state against one norm2 (the
single-read-sweep floor), the expect_paulis route over the full Pauli basis of the kept qubits, and one download to
pinned host memory (what a host-side partial trace starts with).

    python tools/rdm_bench.py OUTDIR [--n 30] [--repeats 5]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Workloads: reduced_density at k = 1, 2, 4, 6, 7, 8 and
10 kept qubits (qubits 0, n-1, then spread over the register); expect_paulis on all 4^k Pauli strings of the same
qubits at k = 2, 4 and 6; one norm2; one download.  Each is the median of the repeats of a host clock around a
synchronising call, after one warm-up.  Reported with the kernel launches, the read sweeps (2^max(0, k-6)) and their
fraction of 3.35 TB/s; the card's name and power limit are read in the same run.  Writes OUTDIR/rdm_bench.json."""
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
from rustqip_b200.state import Context, State, expect_plan  # noqa: E402

PEAK_TBS = 3.35
KS = (1, 2, 4, 6, 7, 8, 10)
PAULI_KS = (2, 4, 6)


def kept(n, k):
    spread = [0, n - 1, 13, 7, 21, 3, 26, 10, 17, 1]
    return [q % n for q in spread[:k]]


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    import torch
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}}
    amp_bytes = 16 << n
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()
            host = torch.empty(amp_bytes, dtype=torch.uint8, pin_memory=True)
            fns = {}
            for k in KS:
                qs = kept(n, k)
                fns["rdm_k%d" % k] = (lambda qs=qs: st.reduced_density(qs), 1 << max(0, k - 6), qs)
            for k in PAULI_KS:
                qs = kept(n, k)
                terms = [[(l, q) for l, q in zip(ls, qs) if l != "I"] for ls in itertools.product("IXYZ", repeat=k)]
                fns["expect_basis_k%d" % k] = (lambda t=terms: st.expect_paulis(t), expect_plan(n, np.complex128, terms),
                                               qs)
            fns["norm2"] = (st.norm2, 1, None)
            fns["download_pinned"] = (lambda: st.download_ptr(host.data_ptr(), 1 << n), 1, None)
            for key, (fn, sweeps, qs) in fns.items():
                fn()  # warm-up
                l0 = ctx.kernel_launches()
                fn()
                launches = ctx.kernel_launches() - l0
                times = [clock(fn) for _ in range(reps)]
                med = float(np.median(times))
                res["workloads"][key] = {"qubits": qs, "sweeps": sweeps, "kernel_launches": launches,
                                         "median_ms": med, "all_ms": times,
                                         "fraction_of_3.35TBs": sweeps * amp_bytes / (med * 1e-3) / (PEAK_TBS * 1e12)}
                print(key, json.dumps(res["workloads"][key]), flush=True)
    w = res["workloads"]
    d = w["norm2"]["median_ms"]
    res["over_norm2"] = {k: v["median_ms"] / d for k, v in w.items()}
    res["rdm_over_expect_basis"] = {k: w["rdm_k%d" % k]["median_ms"] / w["expect_basis_k%d" % k]["median_ms"]
                                    for k in PAULI_KS}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "rdm_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
