"""Time State.sample (qipb200_state_sample) against soft_measure on the N=30 f64 headline state.

    python tools/sample_bench.py OUTDIR [--n 30] [--repeats 5]

Builds the state of the headline circuit (random {H,T,CNOT}, depth 40, seed 0x5EED0002), then times sample for
K = 1, 2^10 and 2^20 seeded draws (every qubit measured, so each result is the drawn index), one soft_measure call,
and one norm2 call (a single read sweep of the state).  Every timed call ends in a stream synchronise, so a host
clock around it is valid; the median of the repeats is reported.  The algorithmic bytes of a sample call are one
read sweep plus the chunks some draw landed in, each read once more.  Writes OUTDIR/sample_bench.json."""
import argparse
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
from rustqip_b200.state import Context, State  # noqa: E402

HBM_BYTES_PER_S = 3.35e12  # H100 SXM data sheet
CHUNK_LOG2 = 12            # amplitudes per chunk of the sampler (kernels.cu: kSampleMaxChunkLog2)


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


def timed(fn, repeats):
    ts, res = [], None
    for _ in range(repeats):
        t0 = time.perf_counter()
        res = fn()
        ts.append((time.perf_counter() - t0) * 1e3)
    return float(np.median(ts)), ts, res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    amp_bytes = 16
    every = list(range(n))[::-1]  # bit i <-> qubit n-1-i <-> index bit i: each result is the drawn index
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "workload": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>"}
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()
            ctx.jit_stats(wait=True)  # no background NVRTC compilation may outlive the process
            # warm-up: first launches, the stream-ordered allocator's pool
            st.sample(every, np.random.default_rng(1).random(1 << 10))
            st.soft_measure([0], 0.5)
            st.norm2()
            res["norm2_ms"], res["norm2_ms_all"], _ = timed(st.norm2, reps)
            res["sample"] = {}
            big = None
            for log_k in (0, 10, 20):
                draws = np.random.default_rng(1000 + log_k).random(1 << log_k)
                l0 = ctx.kernel_launches()
                st.sample(every, draws)
                launches = ctx.kernel_launches() - l0
                ms, all_ms, out = timed(lambda: st.sample(every, draws), reps)
                occupied = int(np.unique(out.astype(np.int64) >> min(CHUNK_LOG2, n)).size)
                nbytes = (amp_bytes << n) + occupied * (amp_bytes << min(CHUNK_LOG2, n))
                res["sample"]["K=2^%d" % log_k] = {
                    "median_ms": ms, "all_ms": all_ms, "kernel_launches": launches, "occupied_chunks": occupied,
                    "algorithmic_bytes": nbytes, "implied_fraction_of_3.35TB/s": nbytes / (ms * 1e-3) / HBM_BYTES_PER_S}
                if log_k == 20:
                    big = (draws, out)
            draws, out = big
            soft_ms, soft_all, _ = timed(lambda: st.soft_measure(every, float(draws[0])), reps)
            agree = [st.soft_measure(every, float(r)) == int(out[k]) for k, r in enumerate(draws[:16])]
    res["soft_measure_ms"], res["soft_measure_ms_all"] = soft_ms, soft_all
    res["soft_measure_agrees_on_16_draws"] = all(agree)
    s = res["sample"]
    res["ratio_sample_2^20_over_soft_measure"] = s["K=2^20"]["median_ms"] / soft_ms
    res["ratio_sample_1_over_soft_measure"] = s["K=2^0"]["median_ms"] / soft_ms
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "sample_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    if not all(agree):
        sys.exit("sample and soft_measure disagree on %d of 16 draws" % agree.count(False))


if __name__ == "__main__":
    main()
