"""Network resets (b200sac_reset): the device time of one reset call, and what periodic resets cost a sampled run.

  python scripts/reset_bench.py [--steps 2000] [--every 200] [--out FILE]

Leg 1: one full reset (every part the handle has, shrink 0) at the bench.py shapes LL, VS, MS, C10 and C10O, and of one
replica of a 64-replica LL handle: 50 calls (about 300 queued operations, within the launch queue) enqueued on one
stream held by a spin kernel (torch.cuda._sleep) until all are queued, so that the CUDA events around them time the
device work alone (the reset kernel, the Adam m / v memsets and the counter write), mean per call; the host's enqueue
time per call is reported beside it.  Leg 2: LunarLander steps/s over --steps sampled steps from a 1 Mi-transition device
ring, with a full reset every --every steps against none; an --every that is not a multiple of 8 also splits the run's
8-step graphs at the boundaries.  The two handles alternate three
times and the median is reported.  The card's name and power limit are read in the same run (nvidia-smi, read-only).
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

from per_bench import card  # noqa: E402


def reset_us(workload, R, calls=50):
    import torch
    from bench import core_config
    from distributed_sac_b200.core import SacCore
    core = SacCore(core_config(workload, R, precision=0 if workload == "LL" else 1), 0, seed=11)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for _ in range(10):
            core.reset(17, replica=0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(1e8))          # ~50 ms of spinning: every call below is queued before e0 fires
        e0.record()
        t0 = time.perf_counter()
        for k in range(calls):
            core.reset(17 + k, replica=R - 1)
        host_us = (time.perf_counter() - t0) * 1e6 / calls
        e1.record()
    e1.synchronize()
    assert e0.elapsed_time(e1) * 1e3 < host_us * calls, "the spin ended before the calls were queued"
    arena_mb = core.arena_floats * 4 / 1e6
    core.close()
    return e0.elapsed_time(e1) * 1e3 / calls, host_us, arena_mb


def run_ms(steps, warmup, every):
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    from bench import core_config
    core = SacCore(core_config("LL", 1, precision=0), 0, seed=11)
    ring = Replay(core, 1 << 20, seed=3)
    ring.fill_synthetic(1 << 20, seed=5)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        core.prepare(ring)
        core.step_sampled(ring, warmup)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        done = 0
        while done < steps:
            n = min(steps - done, every or steps)
            core.step_sampled(ring, n)
            done += n
            if every and done < steps:
                core.reset(1000 + done)
        e1.record()
    e1.synchronize()
    assert torch.isfinite(core.read_losses(64)).all()
    ring.close()
    core.close()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=2000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--every", type=int, default=200)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("reset_bench.py needs a CUDA device")
    res = {"card": card(), "reset_us": {}, "steps": args.steps, "every": args.every}
    for name, wl, R in (("LL", "LL", 1), ("VS", "VS", 1), ("MS", "MS", 1), ("C10", "C10", 1), ("C10O", "C10O", 1),
                        ("LL_R64_one_replica", "LL", 64)):
        us, host, mb = reset_us(wl, R)
        res["reset_us"][name] = {"device_us_per_call": us, "host_us_per_call": host, "arena_MB_per_replica": mb}
        print(json.dumps({name: res["reset_us"][name]}), flush=True)
    base, sched = [], []
    for _ in range(3):
        base.append(run_ms(args.steps, args.warmup, 0))
        sched.append(run_ms(args.steps, args.warmup, args.every))
    b, s = statistics.median(base), statistics.median(sched)
    res["LL_sampled"] = {"no_reset_steps_per_s": 1e3 / b, "reset_steps_per_s": 1e3 / s, "slowdown": s / b,
                         "no_reset_ms": base, "reset_ms": sched}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[reset_bench] {time.time() - t0:.0f} s", file=sys.stderr)
