"""Time State.apply_function (qipb200_state_apply_function) on an N=30 f64 state against the floor of one read-write
sweep measured in the same process.

    python tools/function_bench.py OUTDIR [--n 30] [--repeats 10]

State: H on every qubit from |0>, then rz on every qubit (angles seeded).  Qubit q is index bit n-1-q, so qubits
0..19 are the 20 high index bits and 20..29 the 10 low ones.  Workloads:
  (a) phase only, 20 in-qubits (qubits 5..24), theta seeded: tile path, a 16 MiB phase table;
  (b) Shor-type: x = the 20 high bits, y = the 10 low bits, f(x) = 2^x mod 1007: tile path;
  (c) x = the 20 low bits, y = the 10 high bits, f random: pair path;
  (d) f(x) = A x over GF(2) (random 10 x 20 A, seed 7), x high, y low: tile path, against apply_schedule (fused) of
      its CNOT network; the two results must be bit-identical (max_abs_diff == 0 on the device);
  (e) Function() creation (validation, host tables, upload) at n_in = 20 and 24, with theta.
The floor is apply_pauli_rotations of one single-qubit Z term: exactly one read-write sweep.  Each time is the median
of the repeats of CUDA events recorded on the library's stream around one call, after two warm-up calls (function
creation: a host clock, the call synchronises).  The card's name and power limit are read in the same run.  Writes
OUTDIR/function_bench.json."""
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

import function_ref as fr  # noqa: E402
from rustqip_b200 import gates  # noqa: E402
from rustqip_b200.state import Context, Function, State, function_plan  # noqa: E402


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


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=10)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    import torch  # CUDA events on the library's stream
    rng = np.random.default_rng(30)
    high, low = list(range(0, 20)), list(range(20, n))
    x_high, y_low = high[::-1], low[::-1]
    A = fr.random_matrix(10, 20, 7)
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps, "state": "H layer, then seeded rz layer",
           "workloads": {}}
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream_handle())
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule([gates.h(q) for q in range(n)] + [gates.rz(q, float(a))
                                                                 for q, a in enumerate(rng.uniform(-3, 3, n))])
            st.sync()

            def timed(fn):
                fn()
                fn()
                st.sync()
                l0 = ctx.kernel_launches()
                fn()
                st.sync()
                launches = ctx.kernel_launches() - l0
                times = []
                for _ in range(reps):
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    fn()
                    e1.record(stream)
                    e1.synchronize()
                    times.append(float(e0.elapsed_time(e1)))
                return float(np.median(times)), times, launches

            floor, floor_all, floor_k = timed(lambda: st.apply_pauli_rotations([[("Z", n // 2)]], [0.3]))
            res["floor_ms"], res["floor_all_ms"], res["floor_kernels"] = floor, floor_all, floor_k
            res["floor_GBps"] = 2 * 16 * (1 << n) / (floor * 1e-3) / 1e9
            cases = {
                "a_phase_only_20": (list(range(5, 25)), [], None, rng.uniform(-np.pi, np.pi, 1 << 20)),
                "b_shor_modexp": (x_high, y_low, fr.modexp_table(2, 1007, 20), None),
                "c_low_in_high_out": (low[::-1] + high[10:], high[:10], rng.integers(0, 1 << 10, 1 << 20), None),
                "d_linear": (x_high, y_low, fr.linear_table(A), None),
            }
            for k, (in_q, out_q, f, theta) in cases.items():
                path, tb = function_plan(n, np.complex128, in_q, out_q)
                with Function(ctx, len(in_q), len(out_q), f=f, theta=theta) as fn:
                    med, all_ms, launches = timed(lambda: st.apply_function(fn, in_q, out_q))
                res["workloads"][k] = {"n_in": len(in_q), "n_out": len(out_q), "path": ["tile", "pair"][path],
                                       "tile_bits": tb, "kernels": launches, "ms": med, "all_ms": all_ms,
                                       "x_floor": med / floor}
            # (d) against the CNOT network, and bit-identical results
            ops = fr.cnot_network(A, x_high, y_low)
            dmed, dall, dk = timed(lambda: st.apply_schedule(ops))
            d = res["workloads"]["d_linear"]
            d.update({"network_cnots": len(ops), "network_kernels": dk, "network_ms": dmed, "network_all_ms": dall,
                      "speedup": dmed / d["ms"]})
            st.set_basis(0)
            st.apply_schedule([gates.h(q) for q in range(n)] + [gates.t(q) for q in range(0, n, 3)])
            with State(n, np.complex128, ctx) as other:
                other.set_basis(0)
                other.apply_schedule([gates.h(q) for q in range(n)] + [gates.t(q) for q in range(0, n, 3)])
                with Function(ctx, 20, 10, f=fr.linear_table(A)) as fn:
                    st.apply_function(fn, x_high, y_low)
                other.apply_schedule(ops)
                d["max_abs_diff_vs_network"] = other.max_abs_diff(st)
        # (e) creation
        for n_in in (20, 24):
            f = rng.integers(0, 1 << 10, 1 << n_in)
            th = rng.uniform(-3, 3, 1 << n_in)
            times = []
            for _ in range(3):
                t0 = time.perf_counter()
                Function(ctx, n_in, 10, f=f, theta=th).free()
                times.append((time.perf_counter() - t0) * 1e3)
            res["function_new_ms_n_in_%d" % n_in] = float(np.median(times))
            ctx.release_pool()
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "function_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
