"""Gradient-norm clipping: cost of the grad_clip plan against the default plan, and the in-graph times of its new launches.

  python scripts/clip_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Workloads: LunarLander (1 learner, 1 Mi-transition ring, layer-chained fp32 plan: 4 launches more), MT1 VSAC (1 learner,
128 Ki ring, 400-wide per-layer wgmma plan: 2 more) and 64 LunarLander learners with 8 Ki rings on one GPU (the PBT case).
Each leg alternates three handles three times and reports the median: no grad_clip, grad_clip with +inf thresholds, and
grad_clip with thresholds that bind on every step (0.25 x the norms the handle reported after its warm-up).  The card's
name and power limit are read in the same run (nvidia-smi, read-only query).
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

MODES = ("off", "inf", "binding")


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                     # noqa: BLE001 -- reported, not fatal
        return {"error": repr(e)}


def config(workload, R, grad_clip):
    from distributed_sac_b200.core import CoreConfig
    if workload == "LL":
        return CoreConfig(replicas=R, precision=0, grad_clip=grad_clip)
    return CoreConfig(state_dim=39, act_dim=4, actor_hidden=[400] * 3, critic_hidden=[400] * 3, batch=1024, replicas=R,
                      precision=1, grad_clip=grad_clip)


def leg(workload, R, ring_n, steps, warmup, mode, timeline):
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(config(workload, R, mode != "off"), 0, seed=11)
    ring = Replay(core, ring_n, seed=3)
    ring.fill_synthetic(ring_n, seed=5)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        core.prepare(ring)
        core.step_sampled(ring, warmup)
        if mode == "binding":
            n = core.read_grad_norms(1)[0]
            for r in range(R):
                core.set_grad_clip(critic=0.25 * float(n[r, 0]), actor=0.25 * float(n[r, 1]), replica=r)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        core.step_sampled(ring, steps)
        e1.record()
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / steps
    assert torch.isfinite(core.read_losses(64)[:, :, 0]).all()
    if mode == "binding":
        assert (core.debug("clip")[:2] < 1).all(), "the binding thresholds did not bind"
    tl = None
    if timeline:
        with torch.cuda.stream(stream):
            names = ["sample", "ingest"] + [n for n, _ in core.profile_step(ring, iters=2)][1:]
            t = core.graph_timeline(ring, iters=200)
        torch.cuda.synchronize()
        tl = {"new_launches_us": {f"{i}:{n}": t[i] for i, n in enumerate(names) if n.startswith("grad_norm")
                                  or (mode != "off" and n in ("adam_critic+polyak", "adam_actor", "wgrad{q1,q2}", "wgrad{actor}"))},
              "step_us": sum(t), "all_us": dict(zip(names, t))}
    ring.close()
    core.close()
    return us, tl


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
        raise SystemExit("clip_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "legs": {}}
    for name, wl, R, ring_n in (("LL_1Mi", "LL", 1, 1 << 20), ("VS_128Ki", "VS", 1, 1 << 17), ("LL_x64", "LL", 64, 8192)):
        us = {m: [] for m in MODES}
        tls = {}
        for k in range(3):
            for m in MODES:
                t, tl = leg(wl, R, ring_n, args.steps, args.warmup, m, timeline=(k == 0 and R == 1))
                us[m].append(t)
                if tl is not None:
                    tls[m] = tl
        med = {m: statistics.median(v) for m, v in us.items()}
        out = {"learners": R, "ring_per_learner": ring_n, "us_per_step": med,
               "inf_over_off": med["inf"] / med["off"], "binding_over_off": med["binding"] / med["off"], "runs_us": us}
        if tls:                        # start-to-start times of the unforked timeline run (b200sac_graph_timeline)
            out["graph_timeline"] = tls
        res["legs"][name] = out
        print(json.dumps({name: {k: v for k, v in out.items() if k not in ("runs_us", "graph_timeline")}}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[clip_bench] {time.time() - t0:.0f} s", file=sys.stderr)
