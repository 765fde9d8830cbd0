"""Time State.entanglement_spectrum (qipb200_state_entanglement_spectrum) on the N=30 f64 headline state against its
parts measured in the same run: purity of the same cut (the Gram kernel without the store) or reduced_density of the
side (the s <= 10 route), and torch.linalg.eigvalsh of a random Hermitian 2^s x 2^s complex128 matrix on the device
(the solver's yardstick).

    python tools/spectrum_bench.py OUTDIR [--n 30] [--repeats 3]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0> (as tools/purity_bench.py builds it).  Workloads:
prefix cuts (qubits 0..s-1, the high index bits) at s = 1, 6, 10, 11, 13, a suffix cut (the 13 lowest index bits) and
a scattered side of 13 qubits.  Each time is the median of the repeats of a host clock around a synchronising call,
after one warm-up.  Targets: the call within 1.05 x (purity + eigvalsh) on the Gram route (s >= 11) and within
1.1 x (reduced_density + eigvalsh) for s <= 10; each row says whether its target was met.  The card's name and power
limit are read in the same run.  Writes OUTDIR/spectrum_bench.json."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

from expect_bench import gpu_info  # noqa: E402
from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.state import Context, State, entanglement_spectrum_plan  # noqa: E402


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def timed(fn, reps):
    fn()  # warm-up
    times = [clock(fn) for _ in range(reps)]
    return {"median_ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times)}


def workloads(n):
    rng = np.random.default_rng(13)
    w = {"prefix_s%d" % s: list(range(s)) for s in (1, 6, 10, 11, 13)}
    w["suffix_s13"] = list(range(n - 13, n))
    w["scattered_s13"] = sorted(int(q) for q in rng.permutation(n)[:13])
    return w


def eigvalsh_ms(torch, s, reps):
    """torch.linalg.eigvalsh of a random Hermitian 2^s x 2^s complex128 matrix on the device."""
    K = 1 << s
    g = torch.Generator(device="cuda").manual_seed(s)
    a = torch.randn(K, K, dtype=torch.complex128, device="cuda", generator=g)
    h = (a + a.conj().T) * 0.5
    del a

    def run():
        torch.linalg.eigvalsh(h)
        torch.cuda.synchronize()

    row = timed(run, reps)
    del h
    torch.cuda.empty_cache()
    return row


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=3)
    args = ap.parse_args()
    n, reps = args.n, max(3, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    import torch
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}, "eigvalsh": {}}
    sizes = sorted(set(min(len(qs), n - len(qs)) for qs in workloads(n).values()))
    for s in sizes:  # before the state is allocated
        res["eigvalsh"]["s%d" % s] = eigvalsh_ms(torch, s, reps)
        print("eigvalsh s%d" % s, json.dumps(res["eigvalsh"]["s%d" % s]), flush=True)
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()
            for key, qs in workloads(n).items():
                route, s, kernels, mbytes, loads = entanglement_spectrum_plan(n, np.complex128, qs)
                l0 = ctx.kernel_launches()
                eigs, _, T, S = st._spectrum(qs, False)
                row = {"qubits": qs, "route": route, "s": s, "plan_kernels": kernels, "launches":
                       ctx.kernel_launches() - l0, "matrix_bytes": mbytes, "trace": T, "entropy": S,
                       "lambda_max": float(eigs[0])}
                row["call"] = timed(lambda: st.entanglement_spectrum(qs), reps)
                if route == 2:
                    row["purity"] = timed(lambda: st.purity(qs), reps)
                    part = row["purity"]["median_ms"]
                    factor = 1.05
                else:
                    row["reduced_density"] = timed(lambda: st.reduced_density(qs), reps)
                    part = row["reduced_density"]["median_ms"]
                    factor = 1.1
                ev = res["eigvalsh"]["s%d" % s]["median_ms"]
                row["yardstick_ms"] = part + ev
                row["ratio_to_yardstick"] = row["call"]["median_ms"] / row["yardstick_ms"]
                row["target_ratio"] = factor
                row["target_met"] = row["ratio_to_yardstick"] <= factor
                res["workloads"][key] = row
                print(key, json.dumps(row), flush=True)
    with open(os.path.join(args.outdir, "spectrum_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "ratios": {k: round(v["ratio_to_yardstick"], 4)
                                                    for k, v in res["workloads"].items()}}))


if __name__ == "__main__":
    main()
