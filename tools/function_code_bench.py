"""Time functions given as CUDA source (Function.from_code, qipb200_function_new_code) on an N=30 f64 state against
the floors of one read-write sweep and one read sweep measured in the same process.

    python tools/function_code_bench.py OUTDIR [--n 30] [--repeats 10]

State: H on every qubit from |0>, then rz on every qubit (angles seeded).  Workloads:
  (1) ring MaxCut phase e^{-i gamma C(x)}, C = the cut count of the n-ring by popcount, x = all n qubits (tile path),
      against one read-write sweep (apply_pauli_rotations of one Z term, the floor of tools/function_bench.py) and
      apply_pauli_rotations of the n ZZ terms (the same op up to a global phase);
  (2) Shor-type 2^x mod 1007, x = the 20 high bits, y = the 10 low bits, f computed per index (square-and-multiply
      over a constant table), against the table handle of tools/function_bench.py; the two results must be
      bit-identical (max_abs_diff == 0 on the device);
  (3) expect_function of the ring cost against one read sweep (norm2) and expect_paulis of the n ZZ terms;
  (4) the NVRTC compile of a new program (host clock), and the same program from QIPB200_JIT_CACHE_DIR in a new
      process;
  (5) the kernels that check f over every x (at creation) and theta over every x (at creation and in set_params) at
      n_in = 30, from torch.profiler, and set_params as a whole (CUDA events; it synchronises).
Each time is the median of the repeats of CUDA events recorded on the library's stream around one call, after two
warm-up calls.  The card's name and power limit are read in the same run.  Writes OUTDIR/function_code_bench.json."""
import argparse
import json
import os
import subprocess
import sys
import tempfile
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)

import function_code_ref as fc  # noqa: E402
import function_ref as fr  # noqa: E402
from rustqip_b200 import gates  # noqa: E402
from rustqip_b200.state import Context, Function, State, function_code_compile, function_plan  # noqa: E402


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


def modexp_source(a, N, m):
    """f(x) = a^x mod N over m bits of x: the product of a^(2^i) mod N over the set bits of x."""
    tab = [pow(a, 1 << i, N) for i in range(m)]
    return ("__device__ const uint32_t qip_pow2[%d] = {%s};\n"
            "__device__ uint64_t qip_f(uint64_t x) {\n"
            "  uint32_t r = 1;\n"
            "  for (int i = 0; i < %d; ++i)\n"
            "    if ((x >> i) & 1) r = r * qip_pow2[i] %% %du;\n"
            "  return r;\n}\n" % (m, ", ".join(map(str, tab)), m, N))


COMPILE_FROM_DISK = """
import sys, time
sys.path.insert(0, sys.argv[1])
from rustqip_b200.state import function_code_compile
src = open(sys.argv[2]).read()
t0 = time.perf_counter()
function_code_compile(30, 0, src, theta=True, n_params=1)
print((time.perf_counter() - t0) * 1e3)
"""


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
    gamma = 0.61
    x_high, y_low = list(range(0, 20))[::-1], list(range(20, n))[::-1]
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps, "state": "H layer, then seeded rz layer",
           "workloads": {}}
    W = res["workloads"]
    with Context(0) as ctx:
        stream = torch.cuda.ExternalStream(ctx.stream_handle())
        with State(n, np.complex128, ctx) as st:
            prep = [gates.h(q) for q in range(n)] + [gates.rz(q, float(a)) for q, a in enumerate(rng.uniform(-3, 3, n))]
            st.set_basis(0)
            st.apply_schedule(prep)
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
                return {"ms": float(np.median(times)), "all_ms": times, "kernels": launches}

            rw = timed(lambda: st.apply_pauli_rotations([[("Z", n // 2)]], [0.3]))
            rd = timed(st.norm2)
            res["floor_rw_ms"], res["floor_read_ms"] = rw["ms"], rd["ms"]
            res["floor_rw_GBps"] = 2 * 16 * (1 << n) / (rw["ms"] * 1e-3) / 1e9
            res["floor_read_GBps"] = 16 * (1 << n) / (rd["ms"] * 1e-3) / 1e9
            ring = fc.ring_terms(n)
            with Function.from_code(ctx, n, 0, fc.ring_source(n), theta=True, n_params=1) as cut:
                # (1) the ring phase
                cut.set_params([-gamma])
                w = timed(lambda: st.apply_function(cut, list(range(n))))
                w["path"] = ["tile", "pair"][function_plan(n, np.complex128, [0], [])[0]]
                w["x_floor_rw"] = w["ms"] / rw["ms"]
                pr = timed(lambda: st.apply_pauli_rotations(ring, [-gamma] * n))
                w.update({"pauli_rotations_ms": pr["ms"], "pauli_rotations_kernels": pr["kernels"],
                          "speedup_vs_pauli_rotations": pr["ms"] / w["ms"], "target_x_floor": 1.15,
                          "target_met": w["ms"] <= 1.15 * rw["ms"]})
                W["1_ring_maxcut_phase"] = w
                # (3) the ring energy
                cut.set_params([1.0])
                w = timed(lambda: st.expect_function(cut, list(range(n))))
                w["x_floor_read"] = w["ms"] / rd["ms"]
                ep = timed(lambda: st.expect_paulis(ring))
                w.update({"expect_paulis_ms": ep["ms"], "expect_paulis_kernels": ep["kernels"],
                          "speedup_vs_expect_paulis": ep["ms"] / w["ms"], "target_x_floor": 1.25,
                          "target_met": w["ms"] <= 1.25 * rd["ms"]})
                e_code = st.expect_function(cut, list(range(n)))
                e_pauli = float(np.sum((1.0 - st.expect_paulis(ring)) / 2.0))
                w.update({"energy": e_code, "energy_from_expect_paulis": e_pauli})
                W["3_ring_expect"] = w
            # (2) Shor-type modular exponentiation, code against table
            src = modexp_source(2, 1007, 20)
            with Function.from_code(ctx, 20, 10, src) as code, \
                    Function(ctx, 20, 10, f=fr.modexp_table(2, 1007, 20)) as table:
                w = timed(lambda: st.apply_function(code, x_high, y_low))
                t = timed(lambda: st.apply_function(table, x_high, y_low))
                w.update({"path": ["tile", "pair"][function_plan(n, np.complex128, x_high, y_low)[0]],
                          "x_floor_rw": w["ms"] / rw["ms"], "table_ms": t["ms"], "table_x_floor_rw": t["ms"] / rw["ms"],
                          "target_x_floor": 1.15, "target_met": w["ms"] <= 1.15 * rw["ms"]})
                with State(n, np.complex128, ctx) as other:
                    for s in (st, other):
                        s.set_basis(0)
                        s.apply_schedule(prep)
                    st.apply_function(code, x_high, y_low)
                    other.apply_function(table, x_high, y_low)
                    w["max_abs_diff_vs_table"] = other.max_abs_diff(st)
                W["2_shor_modexp"] = w
            # (5) the checks at n_in = 30
            f_src = "__device__ uint64_t qip_f(uint64_t x) { return (x * 0x9E3779B97F4A7C15ull) >> 60; }\n"
            th_src = fc.ring_source(n)
            w = {}
            try:
                from torch.profiler import ProfilerActivity, profile
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    with Function.from_code(ctx, n, 4, f_src + th_src, theta=True, n_params=1) as fn:
                        fn.set_params([0.5])
                    torch.cuda.synchronize()
                for ev in prof.key_averages():
                    if ev.key in ("qip_fn_check_f", "qip_fn_check_theta"):
                        w[ev.key + "_ms"] = ev.device_time_total / 1e3 / ev.count
                        w[ev.key + "_count"] = ev.count
            except Exception as e:  # the profiler is optional here
                w["profiler_error"] = repr(e)
            with Function.from_code(ctx, n, 0, th_src, theta=True, n_params=1) as fn:
                t0 = time.perf_counter()
                fn.set_params([0.25])
                w["set_params_host_ms"] = (time.perf_counter() - t0) * 1e3
                w["set_params"] = timed(lambda: fn.set_params([0.25]))
            W["5_checks_n_in_30"] = w
    # (4) compile: cold in this process, then from the disk cache in a new one
    with tempfile.TemporaryDirectory() as cache:
        os.environ["QIPB200_JIT_CACHE_DIR"] = cache
        src = fc.ring_source(n) + "// %d\n" % time.time_ns()  # a program no cache has seen
        t0 = time.perf_counter()
        function_code_compile(n, 0, src, theta=True, n_params=1)
        cold = (time.perf_counter() - t0) * 1e3
        path = os.path.join(cache, "src.cu")
        with open(path, "w") as f:
            f.write(src)
        out = subprocess.run([sys.executable, "-c", COMPILE_FROM_DISK, ROOT, path], capture_output=True, text=True,
                             env=dict(os.environ), timeout=600)
        disk = float(out.stdout.strip().splitlines()[-1]) if out.returncode == 0 else None
        del os.environ["QIPB200_JIT_CACHE_DIR"]
    W["4_compile"] = {"cold_ms": cold, "from_disk_cache_ms": disk}
    with open(os.path.join(args.outdir, "function_code_bench.json"), "w") as f:
        json.dump(res, f, indent=1)
    print(json.dumps({k: {kk: vv for kk, vv in v.items() if not kk.startswith("all")} if isinstance(v, dict) else v
                      for k, v in W.items()}, indent=1))
    print("floors: rw %.3f ms, read %.3f ms; gpu %s" % (res["floor_rw_ms"], res["floor_read_ms"], res["gpu"]))


if __name__ == "__main__":
    main()
