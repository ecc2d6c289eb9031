"""Critic inference and the priority refresh: device time of a full refresh of a full prioritized ring, and critic_values
rows per second.

  python scripts/refresh_bench.py [--repeats 5] [--out FILE]

Leg 1: b200sac_replay_refresh_priorities over every slot of a full 1 Mi-transition LunarLander ring and a full
128 Ki-transition VSAC-shape ring (bench.py's LL and VS shapes, rows from fill_synthetic), stochastic next actions; each
call timed with CUDA events around it on its stream (the call synchronises, so the events bracket its device work and the
host's slot list), median over --repeats after one warm-up call.  Leg 2: b200sac_critic_values of q1 and q2 on 1 Mi
device-resident rows at both shapes, rows per second, median over --repeats.  The card's name and power limit are read
in the same run (nvidia-smi, read-only).
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

RINGS = {"LL": 1 << 20, "VS": 1 << 17}


def leg(workload, repeats):
    import torch
    from bench import core_config
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(workload, 1, precision=0 if workload == "LL" else 1), 0, seed=11)
    cap = RINGS[workload]
    ring = Replay(core, cap, seed=3, prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6))
    ring.fill_synthetic(cap, seed=5)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)

    def timed(fn):
        out = []
        fn()
        for _ in range(repeats):
            e0.record()
            fn()
            e1.record()
            e1.synchronize()
            out.append(e0.elapsed_time(e1))
        return statistics.median(out)

    refresh_ms = timed(lambda: ring.refresh_priorities(7))
    rows = 1 << 20
    g = torch.Generator(device="cuda").manual_seed(0)
    obs = torch.randn(rows, core.cfg.obs_dim, device="cuda", generator=g)
    act = torch.rand(rows, core.cfg.act_dim, device="cuda", generator=g) * 2 - 1
    values_ms = timed(lambda: core.critic_values(obs, act))
    flop = 2 * sum(i * o for i, o in zip([core.cfg.obs_dim] + list(core.cfg.actor_hidden), list(core.cfg.actor_hidden) +
                                         [2 * core.cfg.act_dim]))
    cin = [core.cfg.obs_dim + core.cfg.act_dim] + list(core.cfg.critic_hidden)
    flop += 4 * 2 * sum(i * o for i, o in zip(cin, list(core.cfg.critic_hidden) + [1]))
    return {"workload": workload, "ring_slots": cap, "chunk_rows": core.critic_values_chunk(),
            "refresh_ms": round(refresh_ms, 3), "refresh_tflops": round(flop * cap / refresh_ms / 1e9, 2),
            "critic_values_rows_per_s": round(rows / values_ms * 1e3)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    res = {"card": card(), "legs": [leg(w, a.repeats) for w in RINGS]}
    print(json.dumps(res))
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
