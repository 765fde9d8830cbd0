"""Time State.apply_kraus_channels (qipb200_state_apply_kraus_channels) on the N=30 f64 headline state, against the
same run's sweeps and against the route through existing calls.

    python tools/kraus_channel_bench.py OUTDIR [--n 30] [--repeats 9]

State: random {H,T,CNOT}, depth 40, seed 0x5EED0002, from |0>.  Layers:
  (a) amplitude damping along X (gamma = 0.01) on all n qubits: 8 groups of 4, 3 and 1 qubits;
  (b) 15 random two-qubit Stinespring channels of 4 operators on the brickwork pairs (2i, 2i + 1): 8 groups;
  (c) 15 noisy CNOTs, CNOT then two_qubit_depolarizing(0.01), on the brickwork pairs: state-independent, no sweep of
      this call's own (the chosen unitaries go through apply_schedule);
  (d) amplitude damping along Z (gamma = 0.01) on all n qubits through this call and through apply_channels: the cost
      of generality.
Sweep times of the same run: norm2 (a read sweep) and a one-term apply_pauli_rotations (a read-write sweep).  The floor
of a layer with r groups is 1 read + r read-write sweeps; the targets are 1.15 x the floor for (a) and (b), and (a) at
least 4 x faster than the existing-call route (per channel: reduced_density of its qubits, the choice on the host,
apply_op of K / sqrt(p)).  Each number is the median of the repeats of a host clock around the call (which
synchronises), after one warm-up; the card's name and power limit are read in the same run.  Writes
OUTDIR/kraus_channel_bench.json."""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools")):
    if p not in sys.path:
        sys.path.insert(0, p)

from channel_bench import existing_route_groups, gpu_info  # noqa: E402
from rustqip_b200 import channels as ch  # noqa: E402
from rustqip_b200 import circuits  # noqa: E402
from rustqip_b200.state import Context, State, kraus_channels_plan  # noqa: E402

H = np.array([[1, 1], [1, -1]], dtype=np.complex128) / np.sqrt(2)
CX = np.array([[1, 0, 0, 0], [0, 1, 0, 0], [0, 0, 0, 1], [0, 0, 1, 0]], dtype=np.complex128)


def stinespring(k, m, rng):
    D = 1 << k
    a = rng.normal(size=(m * D, D)) + 1j * rng.normal(size=(m * D, D))
    q, _ = np.linalg.qr(a)
    return ch.KrausChannel([q[i * D:(i + 1) * D, :] for i in range(m)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("outdir")
    ap.add_argument("--n", type=int, default=30)
    ap.add_argument("--repeats", type=int, default=9)
    args = ap.parse_args()
    n, reps = args.n, max(5, args.repeats)
    os.makedirs(args.outdir, exist_ok=True)
    rng = np.random.default_rng(31)
    xd = ch.KrausChannel([H @ k @ H for k in ch.amplitude_damping(0.01).kraus])
    brick = [[2 * i, 2 * i + 1] for i in range(n // 2)]
    ncx = ch.KrausChannel([CX]).compose(ch.two_qubit_depolarizing(0.01))
    layers = {
        "a_x_damping_all": ([xd] * n, [[q] for q in range(n)], True),
        "b_stinespring_pairs": ([stinespring(2, 4, rng) for _ in brick], brick, True),
        "c_noisy_cnot_pairs": ([ncx] * len(brick), brick, False),
        "d_z_damping_all": ([ch.KrausChannel(ch.amplitude_damping(0.01))] * n, [[q] for q in range(n)], False),
    }
    res = {"gpu": gpu_info(), "n": n, "dtype": "f64", "repeats": reps,
           "state": "random {H,T,CNOT} depth 40 seed 0x5EED0002 from |0>", "layers": {}}
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
            for name, (chans, groups, route) in layers.items():
                plan = kraus_channels_plan(n, np.complex128, chans, groups)
                med, all_ms, launches = timed(lambda: st.apply_kraus_channels(chans, groups, rng=rng))
                floor = (read + plan[0] * rw) if plan[0] else None
                row = {"channels": len(groups), "plan": plan, "kernels": launches, "ms": med, "all_ms": all_ms,
                       "floor_ms": floor, "x_floor": med / floor if floor else None}
                if name[0] in "ab":
                    row["target_x"] = 1.15
                    row["target_met"] = med / floor <= 1.15
                if route:
                    emed, eall, elaunch = timed(lambda: existing_route_groups(st, chans, groups, rng), repeats=3)
                    row.update({"existing_route_ms": emed, "existing_route_all_ms": eall,
                                "existing_route_kernels": elaunch, "speedup_over_existing_route": emed / med})
                if name.startswith("d"):
                    amed, aall, alaunch = timed(lambda: st.apply_channels(ch.amplitude_damping(0.01), list(range(n)),
                                                                          rng=rng))
                    row.update({"apply_channels_ms": amed, "apply_channels_all_ms": aall,
                                "apply_channels_kernels": alaunch, "x_apply_channels": med / amed})
                res["layers"][name] = row
    print(json.dumps(res, indent=1))
    with open(os.path.join(args.outdir, "kraus_channel_bench.json"), "w") as f:
        json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
