"""Cost of the general-noise SDE path (families of examples/sde_noise_families.cuh: G of size d x m, applied as contractions).

Prints one JSON line, on C5's shape (N = 131 072 members, T = 1, dt = 0.01, saveat every step, EulerHeun, Philox noise
regenerated in the reverse pass, shared p, cost dg = 1):
  * each example family with BacksolveAdjoint and with InterpolatingAdjoint: forward and reverse ms of one gradient (CUDA
    events, median of the timed runs);
  * the built-in diagonal sde_lv against its general-form twin sde_lv_general on identical inputs, alternated run by run,
    with both sensealgs: medians and the twin-over-built-in ratios.
Card name and power limit are read in the same run.  Plug-ins are built by __graft_entry__.build(); a missing one is built
here into a temporary directory.

    python bench_sde_noise.py [--n 131072] [--runs 5]
"""
import argparse
import json
import os
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, ROOT)

# family: (u0, p) nominal, the members' u0 perturbed by 5 %
NOMINAL = {"sde_roessler": ([0.75, 0.5], [-1.5, 0.05, 0.2, 0.01]), "sde_mixing": ([0.75, 0.5], [-1.5, 0.05, 0.2, 0.01]),
           "sde_additive": ([0.2, -0.1], [1.0, 0.3]), "sde_nonsquare": ([1.0, 0.8, 0.6], [1.0, 0.1]),
           "sde_scalar": ([0.6, 0.3], [1.01, 0.87]), "sde_lv_general": ([1.0, 1.0], [1.5, 1.0, 3.0, 1.0, 0.1, 0.1]),
           "sde_lv": ([1.0, 1.0], [1.5, 1.0, 3.0, 1.0, 0.1, 0.1])}


def timed(eng, u0, p):
    import torch
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
    ap.add_argument("--n", type=int, default=131072)
    ap.add_argument("--runs", type=int, default=5)
    a = ap.parse_args()
    import torch
    import scimlsensitivity_jl_b200 as b
    import __graft_entry__ as g
    from bench import gpu_identity
    N, T, dt = a.n, 1.0, 0.01
    ts = np.linspace(0.0, T, 101)
    out = {"metric": "sde_noise", "gpu": gpu_identity(0), "N": N, "T": T, "dt": dt, "stepper": "euler_heun", "runs": a.runs}
    with tempfile.TemporaryDirectory() as tmp:
        for struct, name in g.SDE_NOISE_FAMILIES:
            so = os.path.join(ROOT, "examples", f"libb200fam_{name}.so")
            if not os.path.exists(so):
                so = b.build_family_plugin(os.path.join(ROOT, "examples", "sde_noise_families.cuh"), struct, name,
                                           out=os.path.join(tmp, f"libb200fam_{name}.so"), sde=True, noise="general")
            b.register_family(so)
        rng = np.random.default_rng(0)
        inputs = {}
        for fam, (u0n, pn) in NOMINAL.items():
            d = len(u0n)
            u0 = np.asarray(u0n)[:, None] * np.exp(0.05 * rng.standard_normal((d, N)))
            inputs[fam] = (torch.tensor(u0, device="cuda:0"), torch.tensor(pn, dtype=torch.float64, device="cuda:0"))
        inputs["sde_lv_general"] = inputs["sde_lv"]                       # the twins run on identical inputs
        kw = dict(on_device=True, cost=b.AffineCost(0.0, 1.0), seed=20260923)

        def engine(fam, sa):
            eng = b.DeviceEnsemble(fam, sa, "euler_heun", N, ts, (0.0, T), dt, **kw)
            timed(eng, *inputs[fam])                                      # warm-up: module load
            return eng

        fams = {}
        for _, fam in g.SDE_NOISE_FAMILIES:
            fams[fam] = {}
            for sa in ("backsolve", "interpolating"):
                eng = engine(fam, sa)
                runs = [timed(eng, *inputs[fam]) for _ in range(a.runs)]
                eng.close()
                fams[fam][sa] = {"fwd_ms": float(np.median([r[0] for r in runs])), "rev_ms": float(np.median([r[1] for r in runs]))}
        out["families"] = fams
        twins = {}
        for sa in ("backsolve", "interpolating"):
            engs = {fam: engine(fam, sa) for fam in ("sde_lv", "sde_lv_general")}
            res = {fam: [] for fam in engs}
            for _ in range(a.runs):
                for fam, eng in engs.items():
                    res[fam].append(timed(eng, *inputs[fam]))
            for eng in engs.values():
                eng.close()
            med = {fam: (float(np.median([r[0] for r in v])), float(np.median([r[1] for r in v]))) for fam, v in res.items()}
            twins[sa] = {fam: {"fwd_ms": m[0], "rev_ms": m[1]} for fam, m in med.items()}
            twins[sa]["general_over_builtin"] = {"fwd": med["sde_lv_general"][0] / med["sde_lv"][0],
                                                 "rev": med["sde_lv_general"][1] / med["sde_lv"][1]}
        out["lv_twins"] = twins
    print(json.dumps(out))


if __name__ == "__main__":
    main()
