"""Checkpointed save intervals against the full dense forward solution on bench.py's C1 ensemble (Lotka-Volterra, 65 536
members, InterpolatingAdjoint, adaptive Tsit5 at 1e-8, T = 10, 101 save times, loss = sum(sol), shared p).

Both modes run alternated in one process: full storage at max_steps = 512 (bench.py's setting) and B200ADJ_FLAG_CHECKPOINT_SAVES
at max_steps = 64 per save interval.  Prints one JSON line: median forward / reverse ms over --reps rounds, device_bytes of
each handle, whether the two gradients are bitwise equal, and the card's name and power limit.

    python bench_t5a_checkpointing.py [--members 65536] [--reps 5]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True, text=True, timeout=30)
        name, power = [x.strip() for x in out.stdout.strip().splitlines()[0].split(",")]
        return name, power
    except Exception as e:                      # the measurement still stands; say why the card is unnamed
        import torch
        return torch.cuda.get_device_name(0), f"unknown ({type(e).__name__})"


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--members", type=int, default=65536)
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    import torch
    import scimlsensitivity_jl_b200 as b
    if not torch.cuda.is_available():
        raise SystemExit("bench_t5a_checkpointing.py measures on the GPU; no CUDA device is visible")
    N, T, tol = args.members, 10.0, 1e-8
    saveat = np.linspace(0.0, T, 101)
    u0 = torch.tensor(np.exp(0.2 * np.random.default_rng(3000).standard_normal((2, N))), device="cuda:0")
    p = torch.tensor([1.5, 1.0, 3.0, 1.0], dtype=torch.float64, device="cuda:0")
    modes = {"full": dict(max_steps=512), "checkpointed": dict(max_steps=64, checkpoint_saves=True)}
    engs = {m: b.DeviceEnsemble("lv", "interpolating", "tsit5_adaptive", N, saveat, (0.0, T), 0.0, cost=b.AffineCost(0.0, 1.0),
                                on_device=True, abstol=tol, reltol=tol, **kw) for m, kw in modes.items()}
    times = {m: {"forward": [], "reverse": []} for m in modes}
    grads = {}

    def timed(fn):
        torch.cuda.synchronize()
        t = time.perf_counter()
        r = fn()
        torch.cuda.synchronize()
        return r, 1e3 * (time.perf_counter() - t)

    for rep in range(args.reps + 1):                 # round 0 warms up both modes
        for m, e in engs.items():
            (saved, status), tf = timed(lambda: e.forward(u0, p))
            (du0, dp), tr = timed(lambda: e.reverse())
            if rep == 0:
                assert int((status != 0).sum()) == 0, f"{m}: members stopped early"
                grads[m] = (saved.cpu().numpy(), du0.cpu().numpy(), dp.cpu().numpy())
            else:
                times[m]["forward"].append(tf); times[m]["reverse"].append(tr)
    name, power = card()
    out = {"workload": "C1-ensemble LV d=2 P=4 N=%d InterpolatingAdjoint adaptive Tsit5 tol 1e-8 T=10 saveat=0.1 sum(sol) shared p" % N,
           "gpu": name, "power_limit": power, "reps": args.reps,
           "bitwise_equal": all(np.array_equal(a, c) for a, c in zip(grads["full"], grads["checkpointed"]))}
    for m, e in engs.items():
        out[m] = {"max_steps": modes[m]["max_steps"], "device_bytes": e.device_bytes(),
                  "forward_ms": float(np.median(times[m]["forward"])), "reverse_ms": float(np.median(times[m]["reverse"])),
                  "forward_ms_all": [round(x, 3) for x in times[m]["forward"]], "reverse_ms_all": [round(x, 3) for x in times[m]["reverse"]]}
        e.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
