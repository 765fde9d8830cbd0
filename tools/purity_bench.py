"""Time State.purity (qipb200_state_purity) on the N=30 f64 headline state against a cuBLAS DGEMM rate measured in the
same run, reduced_density (the route below the switch) and one download to pinned host memory (the entry cost of a
host-side purity).

    python tools/purity_bench.py OUTDIR [--n 30] [--repeats 3]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Workloads: prefix cuts (qubits 0..s-1, the high index
bits) at s = 1, 6, 10, 11, 13, 15, so that s = 10 / 11 put one workload on each side of the route switch; a suffix cut
(the s lowest index bits) at s = 15; a scattered side of 13 qubits; reduced_density of qubits 0..9.  Each is the median
of the repeats of a host clock around a synchronising call, after one warm-up.  The DGEMM rate is torch.matmul of two
float64 8192 x 8192 matrices (median of 5 after 2 warm-ups), taken and freed before the state is allocated.  Columns:
the flop count 2^(n+s+2) of the Gram route (4 real products per entry of the upper triangle of G, 2 flops each) and
its fraction of the DGEMM rate; the panel traffic of the Gram kernel, with each block's 64-row panel read from HBM and
the 128-row panel of its block row read once (shared in L2 by co-resident CTAs), and its time at 3.35 TB/s.  The card's
name and power limit are read in the same run.  Writes OUTDIR/purity_bench.json."""
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
from rustqip_b200.state import Context, State, purity_plan  # noqa: E402

PEAK_TBS = 3.35


def clock(fn):
    t0 = time.perf_counter()
    fn()
    return (time.perf_counter() - t0) * 1e3


def dgemm_tflops(torch):
    a = torch.randn(8192, 8192, dtype=torch.float64, device="cuda")
    b = torch.randn(8192, 8192, dtype=torch.float64, device="cuda")
    for _ in range(2):
        torch.matmul(a, b)
    torch.cuda.synchronize()
    ts = []
    for _ in range(5):
        t0 = time.perf_counter()
        torch.matmul(a, b)
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    del a, b
    torch.cuda.empty_cache()
    return 2 * 8192 ** 3 / statistics.median(ts) / 1e12


def workloads(n):
    rng = np.random.default_rng(13)
    w = {"prefix_s%d" % s: list(range(s)) for s in (1, 6, 10, 11, 13, 15)}
    w["suffix_s15"] = list(range(n - 15, n))
    w["scattered_s13"] = sorted(int(q) for q in rng.permutation(n)[:13])
    return w


def panel_bytes(n, s, amp):
    """HBM bytes of the Gram kernel's panels: 64 rows per block, plus 128 rows once per block row."""
    nr = 1 << (s - 7)
    inner = 1 << (n - s)
    return (nr * (nr + 1) * 64 + nr * 128) * inner * amp


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
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "workloads": {}}
    res["dgemm_tflops"] = dgemm_tflops(torch)
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()
            host = torch.empty(16 << n, dtype=torch.uint8, pin_memory=True)
            fns = {key: (lambda qs=qs: st.purity(qs), qs) for key, qs in workloads(n).items()}
            fns["reduced_density_k10"] = (lambda: st.reduced_density(list(range(10))), None)
            fns["download_pinned"] = (lambda: st.download_ptr(host.data_ptr(), 1 << n), None)
            for key, (fn, qs) in fns.items():
                fn()  # warm-up
                l0 = ctx.kernel_launches()
                fn()
                launches = ctx.kernel_launches() - l0
                times = [clock(fn) for _ in range(reps)]
                row = {"median_ms": statistics.median(times), "min_ms": min(times), "max_ms": max(times),
                       "launches": launches}
                if qs is not None:
                    route, s, kernels, blocks = purity_plan(n, np.complex128, qs)
                    row.update({"qubits": qs, "route": route, "s": s, "plan_kernels": kernels, "gram_blocks": blocks,
                                "purity": st.purity(qs)})
                    if route == 2:
                        flops = 2.0 ** (n + s + 2)
                        bts = panel_bytes(n, s, 16)
                        row.update({"flops": flops, "tflops": flops / (row["median_ms"] * 1e-3) / 1e12,
                                    "fraction_of_dgemm": flops / (row["median_ms"] * 1e-3) / 1e12 / res["dgemm_tflops"],
                                    "flop_bound_ms_at_dgemm": flops / (res["dgemm_tflops"] * 1e12) * 1e3,
                                    "panel_bytes": bts, "panel_bound_ms": bts / (PEAK_TBS * 1e12) * 1e3})
                res["workloads"][key] = row
                print(key, json.dumps(row), flush=True)
    res["s10_minus_reduced_density_ms"] = (res["workloads"]["prefix_s10"]["median_ms"]
                                           - res["workloads"]["reduced_density_k10"]["median_ms"])
    with open(os.path.join(args.outdir, "purity_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({"gpu": res["gpu"], "dgemm_tflops": res["dgemm_tflops"],
                      "s10_minus_reduced_density_ms": res["s10_minus_reduced_density_ms"]}))


if __name__ == "__main__":
    main()
