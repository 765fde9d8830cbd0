"""Time State.apply_channels (qipb200_state_apply_channels) and State.apply_multiqubit_channels
(qipb200_state_apply_multiqubit_channels) on the N=30 f64 headline state, against the same run's sweeps and against
the route through existing calls.

    python tools/channel_bench.py OUTDIR [--n 30] [--repeats 5]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Layers:
  (a) amplitude damping, gamma = 0.01, on all n qubits (sample, weight and apply sweeps);
  (b) depolarizing, p = 0.01, on all n qubits, with the draws forced so that qubit 0 takes a Pauli error and every
      other qubit the identity (no sample, no weight: one read-write sweep);
  (c) reset of qubits 0..9 (sample, weight and apply sweeps);
  (d) two_qubit_depolarizing(0.01) on the 15 brickwork pairs (2i, 2i + 1), draws forced so that the last pair takes
      an error and every other pair the identity (one read-write sweep, the pair folded into a byte table);
  (e) two_qubit_depolarizing(0.01) on the pairs (2i, 2i + 1) of qubits 0..19 and amplitude damping (0.01) on qubits
      20..29 (sample, weight and apply sweeps);
  (f) two_qubit_depolarizing(0.01) on the 15 pairs (q, q + 15), every pair forced to an error, so each needs a
      gathered table (one read-write sweep with 15 gathered-table products per amplitude).
Sweep times of the same run: norm2 (a read sweep) and a one-term apply_pauli_rotations (a read-write sweep).  A layer
that samples makes two full read sweeps (the sample's chunk sums and the weight) and one read-write sweep: the target
is 1.25 x their sum; (b) targets 1.1 x one read-write sweep, (d) and (f) 1.25 x.  The existing-call route, per
channel: reduced_density of its qubits, the choice on the host, then apply_op of K / sqrt(p).  Each number is the
median of the repeats (at least 9 for d-f) of a host clock around the call (which synchronises), after one warm-up;
the card's name and power limit are read in the same run.  Writes OUTDIR/channel_bench.json."""
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

from rustqip_b200 import channels as ch  # noqa: E402
from rustqip_b200 import circuits, gates  # noqa: E402
from rustqip_b200.state import Context, State, channels_plan, multiqubit_channels_plan  # noqa: E402


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


def existing_route(st, chan, qubits, rng):
    """Per channel: reduced_density of its qubit, the Born choice on the host, apply_op of K / sqrt(p)."""
    for q in qubits:
        rho = st.reduced_density([q])
        p = np.array([np.real(np.trace(k @ rho @ k.conj().T)) for k in chan.kraus])
        i = min(int(np.searchsorted(np.cumsum(p), rng.random() * p.sum(), side="right")), len(p) - 1)
        st.apply_op(gates.mat([q], list((chan.kraus[i] / np.sqrt(p[i])).reshape(-1))))
    st.sync()


def existing_route_groups(st, chans, groups, rng):
    """existing_route for channels on qubit groups (the first qubit the top bit of the channel's matrices)."""
    for chan, g in zip(chans, groups):
        rho = st.reduced_density(g[::-1])  # bit i of rho's index is g[::-1][i]: the matrix convention
        p = np.maximum(np.array([np.real(np.trace(k @ rho @ k.conj().T)) for k in chan.kraus]), 0.0)
        i = min(int(np.searchsorted(np.cumsum(p), rng.random() * p.sum(), side="right")), len(p) - 1)
        st.apply_op(gates.mat(g, list((chan.kraus[i] / np.sqrt(p[i])).reshape(-1))))
    st.sync()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    layers = {
        "a_amplitude_damping_all": (ch.amplitude_damping(0.01), list(range(n)), None),
        "b_depolarizing_all_forced": (ch.depolarizing(0.01), list(range(n)), [0.5, 0.999] + [0.5] * (n - 1)),
        "c_reset_10": (ch.reset(), list(range(10)), None),
    }
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "layers": {}}
    rng = np.random.default_rng(31)
    dep2, ad = ch.two_qubit_depolarizing(0.01), ch.amplitude_damping(0.01)
    brick = [[2 * i, 2 * i + 1] for i in range(n // 2)]
    far = [[q, q + n // 2] for q in range(n // 2)]
    multi = {
        "d_two_qubit_depolarizing_brickwork_forced": ([dep2] * len(brick), brick,
                                                      [0.5] * len(brick) + [0.999]),
        "e_depolarizing_pairs_and_damping": ([dep2] * 10 + [ad] * (n - 20),
                                             brick[:10] + [[q] for q in range(20, n)], None),
        "f_gathered_pairs_forced": ([dep2] * len(far), far, [0.5] + [0.999] * len(far)),
    }
    with Context(0) as ctx:
        with State(n, np.complex128, ctx) as st:
            st.set_basis(0)
            st.apply_schedule(circuits.random_circuit(n, 40, 0x5EED0002, "H,T,CNOT"))
            st.sync()

            def timed(fn, repeats=reps):
                fn()  # warm-up
                st.sync()
                l0 = ctx.kernel_launches()
                fn()
                st.sync()
                launches = ctx.kernel_launches() - l0
                times = []
                for _ in range(repeats):
                    t0 = time.perf_counter()
                    fn()
                    st.sync()
                    times.append((time.perf_counter() - t0) * 1e3)
                return float(np.median(times)), times, launches

            read, read_all, _ = timed(st.norm2)
            rw, rw_all, _ = timed(lambda: st.apply_pauli_rotations([[("X", 0)]], [0.1]))
            res["read_sweep_ms"], res["read_sweep_all_ms"] = read, read_all
            res["rw_sweep_ms"], res["rw_sweep_all_ms"] = rw, rw_all
            for name, (chan, qubits, draws) in layers.items():
                plan = channels_plan(n, np.complex128, chan, qubits)
                med, all_ms, launches = timed(lambda: st.apply_channels(chan, qubits, rng=rng, draws=draws))
                sweeps_ms = (2 * read + rw) if plan[0] else rw
                target = 1.25 if plan[0] else 1.1
                emed, eall, elaunch = timed(lambda: existing_route(st, chan, qubits, rng), repeats=3)
                res["layers"][name] = {
                    "channels": len(qubits), "plan": plan, "kernels": launches, "ms": med, "all_ms": all_ms,
                    "sweeps_ms": sweeps_ms, "x_sweeps": med / sweeps_ms, "target_x": target,
                    "target_met": med / sweeps_ms <= target,
                    "existing_route_ms": emed, "existing_route_all_ms": eall, "existing_route_kernels": elaunch,
                    "speedup_over_existing_route": emed / med}
            for name, (chans, groups, draws) in multi.items():
                plan = multiqubit_channels_plan(n, np.complex128, chans, groups)
                med, all_ms, launches = timed(
                    lambda: st.apply_multiqubit_channels(chans, groups, rng=rng, draws=draws), repeats=max(9, reps))
                sweeps_ms = (2 * read + rw) if plan[0] else rw
                emed, eall, elaunch = timed(lambda: existing_route_groups(st, chans, groups, rng), repeats=3)
                res["layers"][name] = {
                    "channels": len(groups), "plan": plan, "kernels": launches, "ms": med, "all_ms": all_ms,
                    "sweeps_ms": sweeps_ms, "x_sweeps": med / sweeps_ms, "target_x": 1.25,
                    "target_met": med / sweeps_ms <= 1.25,
                    "existing_route_ms": emed, "existing_route_all_ms": eall, "existing_route_kernels": elaunch,
                    "speedup_over_existing_route": emed / med}
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "channel_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
