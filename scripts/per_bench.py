"""Prioritized vs uniform replay on the device ring: steps/s of the sampled step and the in-graph times of the two PER
kernels.

  python scripts/per_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Workloads: LunarLander (1 learner, 1 Mi-transition ring, layer-chained fp32 plan), MT1 VSAC (1 learner, 400-wide wgmma
plan) and 64 LunarLander learners on one GPU.  Each leg alternates uniform and prioritized handles three times and reports
the median.  The card's name and power limit are read in the same run (nvidia-smi, read-only query).
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

PER = dict(alpha=0.6, beta=0.4, eps=1e-6)


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


def leg(workload, R, ring_n, steps, warmup, prioritized):
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    cfg, _ = config(workload, R)
    core = SacCore(cfg, 0, seed=11)
    ring = Replay(core, ring_n, seed=3, prioritized=prioritized)
    ring.fill_synthetic(ring_n, seed=5)
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
    tl = None
    if prioritized is not None and R == 1:
        with torch.cuda.stream(stream):
            names = [n for n, _ in core.profile_step(ring, iters=2)]
            tl = core.graph_timeline(ring, iters=200)
        torch.cuda.synchronize()
        # timeline order: per_sample, ingest, the plan's launches with per_update right after the critic-loss launch
        j = next(i for i, n in enumerate(names) if n in ("critic_heads", "chain2{qt->y->bwd q}"))
        tl = {"per_sample_us": tl[0], "per_update_us": tl[j + 2], "all_us": tl, "plan": names[1:]}
    ring.close()
    core.close()
    return ms, tl


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("per_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "per": PER, "legs": {}}
    for name, wl, R, ring_n in (("LL_1Mi", "LL", 1, 1 << 20), ("VS", "VS", 1, 1 << 17), ("LL_x64", "LL", 64, 8192)):
        uni, per, tl = [], [], None
        for _ in range(3):
            uni.append(leg(wl, R, ring_n, args.steps, args.warmup, None)[0])
            ms, t = leg(wl, R, ring_n, args.steps, args.warmup, PER)
            per.append(ms)
            tl = t or tl
        u, p = statistics.median(uni), statistics.median(per)
        out = {"learners": R, "ring_per_learner": ring_n,
               "uniform_steps_per_s": R * 1e3 / u, "per_steps_per_s": R * 1e3 / p, "per_over_uniform": u / p,
               "uniform_ms": uni, "per_ms": per}
        if tl is not None:            # start-to-start times of the unforked timeline run (b200sac_graph_timeline)
            out["graph_timeline"] = tl
        res["legs"][name] = out
        print(json.dumps({name: {k: v for k, v in out.items() if not k.endswith("_ms")}}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[per_bench] {time.time() - t0:.0f} s", file=sys.stderr)
