"""Update intervals on the device ring: steps/s of the sampled step at actor_every in {1, 2, 4} x target_every in {1, 2}.

  python scripts/interval_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Workloads: LunarLander (1 learner, 1 Mi-transition ring, layer-chained fp32 plan) and MT1 VSAC (1 learner, 400-wide
wgmma per-layer plan).  A critic-only step skips the actor update's launches (3 of the 7 critical-path launches of the
chained plan; phases D and E of the per-layer plan), so its gain depends on the plan.  Each schedule's leg alternates
with a default-schedule handle three times and reports the median.  The card's name and power limit are read in the same
run (nvidia-smi, read-only query).
"""
import argparse
import json
import os
import statistics
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "scripts"))

from per_bench import card, config  # noqa: E402

SCHEDULES = [(a, t) for a in (1, 2, 4) for t in (1, 2)]


def leg(workload, ring_n, steps, warmup, actor_every, target_every):
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    cfg, _ = config(workload, 1)
    core = SacCore(cfg, 0, seed=11)
    core.set_update_intervals(actor_every, target_every)
    ring = Replay(core, ring_n, seed=3)
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
    assert torch.isfinite(core.read_losses(64)[:, :, 0]).all()      # (actor-side entries are NaN on critic-only steps)
    ring.close()
    core.close()
    return ms


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
        raise SystemExit("interval_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "legs": {}}
    for name, wl, ring_n in (("LL_1Mi", "LL", 1 << 20), ("VS", "VS", 1 << 17)):
        for a, t in SCHEDULES:
            base, sched = [], []
            for _ in range(3):
                base.append(leg(wl, ring_n, args.steps, args.warmup, 1, 1))
                sched.append(leg(wl, ring_n, args.steps, args.warmup, a, t))
            b, s = statistics.median(base), statistics.median(sched)
            out = {"actor_every": a, "target_every": t, "default_steps_per_s": 1e3 / b, "steps_per_s": 1e3 / s,
                   "speedup": b / s, "default_ms": base, "ms": sched}
            res["legs"][f"{name}_a{a}_t{t}"] = out
            print(json.dumps({f"{name}_a{a}_t{t}": {k: v for k, v in out.items() if not k.endswith("ms")}}), flush=True)
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[interval_bench] {time.time() - t0:.0f} s", file=sys.stderr)
