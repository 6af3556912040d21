"""Cost of the family-event path (VectorContinuousCallback with the conditions and affect compiled into a family plug-in).

Prints one JSON line:
  * projectile: 65 536 ProjectileWall members (examples/vector_callback_families.cuh: floor and wall, both reflecting) with
    perturbed u0 and per-member p, GaussAdjoint, abstol = reltol = 1e-10, saveat 0.5 on [0, 10]: forward and reverse ms
    (CUDA events, median of the timed runs) and trajectories / s of one gradient;
  * ball: the built-in `ball` with its named ContinuousCallback against the BallEvents plug-in (the same callback as family
    conditions) on identical inputs, alternated, 3 runs each.
Card name and power limit are read in the same run.  Plug-ins are built by __graft_entry__.build(); a missing one is built
here into a temporary directory.

    python bench_family_events.py [--n 65536] [--runs 3]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)


def plugin(b, struct, name, tmp):
    header = os.path.join(ROOT, "examples", "vector_callback_families.cuh")
    so = os.path.join(ROOT, "examples", f"libb200fam_{name}.so")
    if not os.path.exists(so):
        so = b.build_family_plugin(header, struct, name, out=os.path.join(tmp, f"libb200fam_{name}.so"), has_events=True)
    b.register_family(so)
    return name


def timed(eng, u0, p, check=False):
    import torch
    if check:                                                        # warm-up: module load, block-size choice, status
        _, st = eng.forward(u0, p)
        assert int((st != 0).sum()) == 0, ("a member did not finish (status 2: max_steps, 3: max_events)", np.bincount(st.cpu().numpy()))
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    ev[0].record()
    eng.forward(u0, p, want_status=False)
    ev[1].record()
    eng.reverse()
    ev[2].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])


def main():
    ap = argparse.ArgumentParser(description=__doc__.split("\n")[0])
    ap.add_argument("--n", type=int, default=65536)
    ap.add_argument("--runs", type=int, default=3)
    a = ap.parse_args()
    import torch
    import scimlsensitivity_jl_b200 as b
    from bench import gpu_identity
    out = {"metric": "family_events", "gpu": gpu_identity(0)}
    with tempfile.TemporaryDirectory() as tmp:
        proj = plugin(b, "ProjectileWall", "projectile", tmp)
        ballev = plugin(b, "BallEvents", "ball_events", tmp)
        N = a.n
        rng = np.random.default_rng(0)
        r = lambda: rng.uniform(-1, 1, N)
        dev = "cuda:0"
        u0 = torch.tensor(np.stack([50.0 + 0.2 * r(), 0.05 * r(), 0.005 * (1 + r()), 2.01 + 0.003 * r()]), device=dev)
        p = torch.tensor(np.stack([9.8 + 0.02 * r(), 0.9 + 0.003 * r()]), device=dev)
        ts = np.arange(0.0, 10.0 + 1e-12, 0.5)
        kw = dict(abstol=1e-10, reltol=1e-10, on_device=True, shared_p=False, cost=b.AffineCost(1.0, -1.0), max_steps=1024)
        eng = b.DeviceEnsemble(proj, "gauss", "tsit5_adaptive", N, ts, (0.0, 10.0), 0.0, **kw)
        eng.set_continuous_callback(b.VectorContinuousCallback(max_events=8))
        timed(eng, u0, p, check=True)
        runs = [timed(eng, u0, p) for _ in range(a.runs)]
        f_ms, r_ms = float(np.median([x[0] for x in runs])), float(np.median([x[1] for x in runs]))
        counts, _ = eng.event_times()
        out["projectile"] = {"N": N, "sensealg": "gauss", "tol": 1e-10, "fwd_ms": f_ms, "rev_ms": r_ms,
                             "traj_per_s": N / ((f_ms + r_ms) * 1e-3), "events_per_member": float(np.mean(counts))}
        del eng
        # named ball against the BallEvents plug-in, identical inputs, alternated
        # (restitution and height kept away from the Zeno limit inside [0, 15]: at most ~10 bounces per member)
        u0b = torch.tensor(np.stack([np.clip(50.0 + 5.0 * rng.standard_normal(N), 40.0, 60.0), 0.5 * rng.standard_normal(N)]), device=dev)
        pb = torch.tensor(np.stack([9.8 + 0.3 * rng.standard_normal(N), np.clip(0.8 + 0.03 * rng.standard_normal(N), 0.75, 0.85)]), device=dev)
        tb = np.linspace(0.5, 15.0, 30)
        kb = dict(abstol=1e-10, reltol=1e-10, on_device=True, shared_p=False, cost=b.AffineCost(1.0, 0.0), max_steps=1024)
        named = b.DeviceEnsemble("ball", "gauss", "tsit5_adaptive", N, tb, (0.0, 15.0), 0.0, **kb)
        named.set_continuous_callback(b.ContinuousCallback(idx=0, direction=-1, p_comp=1, p_param=1, p_sign=-1.0, max_events=16))
        fam = b.DeviceEnsemble(ballev, "gauss", "tsit5_adaptive", N, tb, (0.0, 15.0), 0.0, **kb)
        fam.set_continuous_callback(b.VectorContinuousCallback(direction=-1, max_events=16))
        timed(named, u0b, pb, check=True); timed(fam, u0b, pb, check=True)
        res = {"named": [], "family": []}
        for _ in range(a.runs):
            res["named"].append(timed(named, u0b, pb))
            res["family"].append(timed(fam, u0b, pb))
        summ = {}
        for k, v in res.items():
            summ[k] = {"fwd_ms": [round(x[0], 4) for x in v], "rev_ms": [round(x[1], 4) for x in v]}
        med = {k: (float(np.median(summ[k]["fwd_ms"])), float(np.median(summ[k]["rev_ms"]))) for k in summ}
        summ["family_over_named"] = {"fwd": med["family"][0] / med["named"][0], "rev": med["family"][1] / med["named"][1],
                                     "total": sum(med["family"]) / sum(med["named"])}
        out["ball"] = dict(N=N, sensealg="gauss", **summ)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
