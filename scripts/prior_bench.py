"""Prior-data rings (symmetric sampling): sampled-step rate with a prior attached against the plain ring.

  python scripts/prior_bench.py [--steps 2000] [--rounds 5] [--out FILE]

Per workload (bench.py's LL, VS and MS shapes; precision 0 at LL, 1 otherwise), three handles of the same configuration and
seed, each with an online ring of RING[w] transitions filled by fill_synthetic:
  plain  nothing attached;
  m0     a prior of the same capacity attached, m = 0 (the plain draw through the mixed sampler and gather);
  half   the same, m = P / 2 (P = batch / num_tasks): half of every task block from the prior.
Rate: steps / s of `--steps` pipelined step_sampled calls in 8-step graphs, timed with CUDA events; the three legs
alternate for --rounds rounds after one warm-up round, and the median round of each leg is reported.  In-graph times: the
sampler's and the gather's start-to-start times from b200sac_graph_timeline (one step per graph).  The card's name and
power limit are read in the same run (nvidia-smi, read-only).
"""
import argparse
import json
import os
import statistics
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from per_bench import card  # noqa: E402

RING = {"LL": 1 << 20, "VS": 1 << 17, "MS": 1 << 17}
LEGS = ("plain", "m0", "half")


def workload(w, steps, rounds):
    import torch
    from bench import core_config
    from distributed_sac_b200.core import Replay, SacCore
    cfg = core_config(w, 1, precision=0 if w == "LL" else 1)
    P = cfg.batch // max(cfg.num_tasks, 1)
    legs = {}
    for name in LEGS:
        core = SacCore(cfg, 0, seed=11)
        ring = Replay(core, RING[w], seed=3)
        ring.fill_synthetic(RING[w], seed=5)
        prior = None
        if name != "plain":
            prior = Replay(core, RING[w], seed=4)
            prior.fill_synthetic(RING[w], seed=6)
            ring.attach_prior(prior)
            ring.set_prior_rows(P // 2 if name == "half" else 0)
        core.prepare(ring)
        legs[name] = (core, ring, prior)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    rates = {name: [] for name in LEGS}
    for rnd in range(rounds + 1):
        for name in LEGS:
            core, ring, _ = legs[name]
            e0.record()
            core.step_sampled(ring, steps)
            e1.record()
            e1.synchronize()
            if rnd > 0:
                rates[name].append(steps / (e0.elapsed_time(e1) * 1e-3))
    out = {"workload": w, "ring": RING[w], "prior_rows": {"m0": 0, "half": P // 2}, "P": P}
    for name in LEGS:
        core, ring, _ = legs[name]
        tl = core.graph_timeline(ring, iters=200)
        out[name] = {"steps_per_s": round(statistics.median(rates[name]), 1),
                     "rounds_steps_per_s": [round(x, 1) for x in rates[name]],
                     "sampler_us": round(tl[0], 2), "gather_us": round(tl[1], 2)}
    for core, ring, prior in legs.values():
        ring.close()
        if prior is not None:
            prior.close()
        core.close()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "legs": [workload(w, a.steps, a.rounds) for w in RING]}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
