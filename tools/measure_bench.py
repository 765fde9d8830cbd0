"""Time State.measure (qipb200_state_measure) against soft_measure + measure_prob + collapse on the N=30 f64 headline
state, and the real cost of a mid-circuit measurement: measure followed by the next schedule, minus that schedule.

    python tools/measure_bench.py OUTDIR [--n 30] [--repeats 5]

Builds the state of the headline circuit (random {H,T,CNOT}, depth 40, seed 0x5EED0002) and measures qubit 0 with
seeded draws.  Timed, each as the median of the repeats of a host clock around work that ends in a stream
synchronise:
  (a) soft_measure + measure_prob + collapse, and each of the three on its own;
  (b) measure alone (the collapse it leaves pending is applied, untimed, before the next repeat);
  (c) measure followed by the next 40-layer schedule (seed 0x5EED0006), minus that schedule alone; the two are
      alternated repeat by repeat.
The kernel launches of each are counted, and the card's name and power limit are read in the same run.  Writes
OUTDIR/measure_bench.json."""
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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    q = [0]
    draws = iter(np.random.default_rng(30).random(1000))
    nxt = circuits.random_circuit(n, 40, 0x5EED0006, "H,T,CNOT")
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps, "measured_qubits": q,
           "workload": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>; next schedule: depth 40 seed 0x5EED0006"}
    times = {k: [] for k in ("soft_measure", "measure_prob", "collapse", "three_calls", "measure",
                             "measure_then_schedule", "schedule_alone")}
    launches = {}
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()

            def three():
                m = st.soft_measure(q, next(draws))
                p = st.measure_prob(m, q)
                st.collapse(q, m, p)
                st.sync()

            def measure():
                st.measure(q, next(draws))

            def measure_then_schedule():
                st.measure(q, next(draws))
                st.apply_schedule(nxt)
                st.sync()

            def schedule_alone():
                st.apply_schedule(nxt)
                st.sync()

            # warm-up: first launches, the allocator's pool, and the generated kernels of both schedules (the one that
            # carries the collapse in its first pass differs from the plain one)
            three()
            measure()
            st.norm2()
            measure_then_schedule()
            schedule_alone()
            ctx.jit_stats(wait=True)
            measure_then_schedule()
            schedule_alone()
            for name, fn in (("three_calls", three), ("measure", measure), ("measure_then_schedule", measure_then_schedule),
                             ("schedule_alone", schedule_alone)):
                st.norm2()  # applies a collapse left pending by the previous step, untimed
                l0 = ctx.kernel_launches()
                fn()
                launches[name] = ctx.kernel_launches() - l0
            st.norm2()
            launches["measure_then_schedule_minus_schedule"] = launches["measure_then_schedule"] - launches["schedule_alone"]
            for _ in range(reps):
                m = st.soft_measure(q, next(draws))
                times["soft_measure"].append(clock(lambda: st.soft_measure(q, next(draws))))
                times["measure_prob"].append(clock(lambda: st.measure_prob(m, q)))
                p = st.measure_prob(m, q)
                times["collapse"].append(clock(lambda: (st.collapse(q, m, p), st.sync())))
                times["three_calls"].append(clock(three))
                st.norm2()
                times["measure"].append(clock(measure))
                st.norm2()
                times["measure_then_schedule"].append(clock(measure_then_schedule))
                times["schedule_alone"].append(clock(schedule_alone))
            js = ctx.jit_stats(wait=True)
    med = {k: float(np.median(v)) for k, v in times.items()}
    res["median_ms"] = med
    res["all_ms"] = times
    res["kernel_launches"] = launches
    res["jit"] = js
    res["a_three_calls_ms"] = med["three_calls"]
    res["b_measure_ms"] = med["measure"]
    res["c_measure_in_circuit_ms"] = med["measure_then_schedule"] - med["schedule_alone"]
    res["c_below_b_plus_collapse"] = res["c_measure_in_circuit_ms"] < med["measure"] + med["collapse"]
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "measure_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
