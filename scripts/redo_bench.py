"""Dormant-neuron recycling (b200sac_redo): the device time of one recycle call, and what periodic recycles cost a sampled
run.

  python scripts/redo_bench.py [--steps 4000] [--every 1000] [--out FILE]

Leg 1: one recycle (a batch of rows from the ring, thresholds 0.1 for the actor and the critics, so that the recycle
kernel has neurons to write) at the bench.py shapes LL, VS, MS and C10: 50 calls enqueued on one stream held by a spin
kernel (torch.cuda._sleep) until all are queued, so that the CUDA events around them time the device work alone (the
input copies, the per-layer forward, the score kernel and the recycle kernel), mean per call; the host's enqueue time
per call is reported beside it.  Leg 2: LunarLander steps/s over --steps sampled steps from a 1 Mi-transition device
ring, with a recycle every --every steps (its batch drawn from the ring with Replay.sample(), as the learners draw it)
against none.  The two handles alternate three times and the median is reported.  The card's name and power limit are
read in the same run (nvidia-smi, read-only).
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


def redo_us(workload, calls=50):
    import torch
    from bench import core_config
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(core_config(workload, 1, precision=0 if workload == "LL" else 1), 0, seed=11)
    ring = Replay(core, 1 << 16, seed=3)
    ring.fill_synthetic(1 << 16, seed=5)
    s, a = (t.cuda() for t in ring.sample()[:2])
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        for _ in range(10):
            core.redo(17, s, a, actor=0.1, critic=0.1)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda._sleep(int(1e8))          # ~50 ms of spinning: every call below is queued before e0 fires
        e0.record()
        t0 = time.perf_counter()
        for k in range(calls):
            core.redo(17 + k, s, a, actor=0.1, critic=0.1)
        host_us = (time.perf_counter() - t0) * 1e6 / calls
        assert not e0.query(), "the spin ended before the calls were queued"
        e1.record()
    e1.synchronize()
    neurons = sum(core.cfg.actor_hidden) + 2 * sum(core.cfg.critic_hidden)
    ring.close()
    core.close()
    return e0.elapsed_time(e1) * 1e3 / calls, host_us, neurons


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
                s, a = ring.sample()[:2]
                core.redo(1000 + done, s.cuda(), a.cuda(), actor=0.1, critic=0.1)
        e1.record()
    e1.synchronize()
    assert torch.isfinite(core.read_losses(64)).all()
    ring.close()
    core.close()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=4000)
    ap.add_argument("--warmup", type=int, default=200)
    ap.add_argument("--every", type=int, default=1000)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("redo_bench.py needs a CUDA device")
    res = {"card": card(), "redo_us": {}, "steps": args.steps, "every": args.every}
    for name in ("LL", "VS", "MS", "C10"):
        us, host, neurons = redo_us(name)
        res["redo_us"][name] = {"device_us_per_call": us, "host_us_per_call": host, "hidden_neurons": neurons}
        print(json.dumps({name: res["redo_us"][name]}), flush=True)
    base, sched = [], []
    for _ in range(3):
        base.append(run_ms(args.steps, args.warmup, 0))
        sched.append(run_ms(args.steps, args.warmup, args.every))
    b, s = statistics.median(base), statistics.median(sched)
    res["LL_sampled"] = {"no_redo_steps_per_s": 1e3 / b, "redo_steps_per_s": 1e3 / s, "slowdown": s / b,
                         "no_redo_ms": base, "redo_ms": sched}
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[redo_bench] {time.time() - t0:.0f} s", file=sys.stderr)
