"""n-step returns on the device ring: step time of the sampled step from an unlinked ring and from a linked ring at
n = 1, 3 and 5, and the in-graph time of the gather (the launch that folds the return).

  python scripts/nstep_bench.py [--steps 1000] [--warmup 100] [--out FILE]

Workloads: LunarLander (1 learner, 1 Mi-transition ring, layer-chained fp32 plan), MT1 VSAC (1 learner, 400-wide wgmma
plan) and 64 LunarLander learners on one GPU.  The rings are filled synthetically: a linked ring then chains slot i to
i + 1 (d ~ Bernoulli(0.01)), so nearly every row folds the full horizon.  Each workload alternates the four handles three
times and reports the medians.  The card's name, power limit and SM clock are read in the same run (nvidia-smi, read-only
query).
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

VARIANTS = (("unlinked", None), ("n1", 1), ("n3", 3), ("n5", 5))


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                     # noqa: BLE001 -- reported, not fatal
        return {"error": repr(e)}


def config(workload, R):
    from distributed_sac_b200.core import CoreConfig
    if workload == "LL":
        return CoreConfig(replicas=R, precision=0), 0
    return CoreConfig(state_dim=39, act_dim=4, actor_hidden=[400] * 3, critic_hidden=[400] * 3, batch=1024, replicas=R,
                      precision=1), 1


def leg(workload, R, ring_n, steps, warmup, n_step, timeline):
    """(ms per step, mean hops folded per row, in-graph us of the gather or None) of one fresh handle."""
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    cfg, _ = config(workload, R)
    core = SacCore(cfg, 0, seed=11)
    ring = Replay(core, ring_n, seed=3, trajectories=n_step is not None)
    ring.fill_synthetic(ring_n, seed=5)
    if n_step is not None:
        ring.set_nstep(n_step)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        core.prepare(ring)
        core.step_sampled(ring, warmup)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        core.step_sampled(ring, steps)
        e1.record()
    e1.synchronize()
    ms = e0.elapsed_time(e1) / steps
    assert torch.isfinite(core.read_losses(64)).all()
    hops = None if n_step is None else float(core.debug("nstep_m").float().mean())
    gather = None
    if timeline:
        with torch.cuda.stream(stream):
            gather = core.graph_timeline(ring, iters=200)[1]      # [sample, ingest, plan...]: start of the gather to the next launch
        torch.cuda.synchronize()
    ring.close()
    core.close()
    return ms, hops, gather


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("nstep_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "legs": {}}
    for name, wl, R, ring_n in (("LL_1Mi", "LL", 1, 1 << 20), ("VS", "VS", 1, 1 << 17), ("LL_x64", "LL", 64, 8192)):
        ms = {v: [] for v, _ in VARIANTS}
        hops, gather = {}, {}
        for rnd in range(3):
            for v, n in VARIANTS:
                t, h, g = leg(wl, R, ring_n, args.steps, args.warmup, n, timeline=rnd == 2)
                ms[v].append(t)
                hops[v], gather[v] = h, g
        med = {v: statistics.median(x) for v, x in ms.items()}
        out = {"learners": R, "ring_per_learner": ring_n,
               "step_us": {v: 1e3 * m for v, m in med.items()},
               "steps_per_s": {v: R * 1e3 / m for v, m in med.items()},
               "over_unlinked": {v: m / med["unlinked"] for v, m in med.items()},
               "mean_hops": hops, "gather_us": gather, "all_ms": ms}
        res["legs"][name] = out
        print(json.dumps({name: {k: v for k, v in out.items() if k != "all_ms"}}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[nstep_bench] {time.time() - t0:.0f} s", file=sys.stderr)
