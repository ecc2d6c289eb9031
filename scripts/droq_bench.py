"""Dropout Q-functions (b200sac_cfg.critic_dropout): what drawing and applying the masks costs a sampled step.

  python scripts/droq_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Leg 1: steps/s of sampled steps from a 1 Mi-transition device ring at the bench.py shapes LL (precision 0; one replica and
16 replicas), VS and MS (precision 1, one replica), for three handles of each: the critic_ln handle, and the
critic_dropout handle at p = 0 and at p = 0.01.  The handles alternate three times and the median is reported.  Leg 2:
the device time of every LayerNorm launch of one step of the critic_ln handle and of the p = 0.01 handle
(b200sac_profile_step, CUDA events around each launch of an eager step).  The card's name, power limit and maximum SM
clock are read in the same run (nvidia-smi, read-only).
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

CASES = [("LL", 1, 0), ("LL", 16, 0), ("VS", 1, 1), ("MS", 1, 1)]
KINDS = {"ln": None, "droq_p0": 0.0, "droq_p0.01": 0.01}      # handle -> dropout rate (None: critic_ln only)


def make(workload, R, precision, p):
    from bench import core_config
    from distributed_sac_b200.core import SacCore
    cfg = core_config(workload, R, precision=precision)
    cfg.critic_layer_norm = True
    cfg.critic_dropout = p is not None
    core = SacCore(cfg, 0, seed=11)
    if p is not None:
        core.set_critic_dropout(p)
    return core


def run_ms(core, ring, steps, warmup):
    import torch
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        core.step_sampled(ring, warmup)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        core.step_sampled(ring, steps)
        e1.record()
    e1.synchronize()
    assert torch.isfinite(core.read_losses(16)).all()
    return e0.elapsed_time(e1) / steps


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
        raise SystemExit("droq_bench.py needs a CUDA device")
    from distributed_sac_b200.core import Replay
    res = {"card": card(), "steps": args.steps, "cases": {}}
    for workload, R, precision in CASES:
        name = f"{workload} R={R} precision {precision}"
        handles = {}
        for kind, p in KINDS.items():
            core = make(workload, R, precision, p)
            ring = Replay(core, 1 << 20, "device", seed=3)
            ring.fill_synthetic(1 << 20, seed=5)
            core.prepare(ring)
            handles[kind] = (core, ring)
        times = {k: [] for k in KINDS}
        for _ in range(3):
            for kind in KINDS:
                times[kind].append(run_ms(*handles[kind], args.steps, args.warmup))
        case = {f"{k}_steps_per_s": 1e3 / statistics.median(times[k]) for k in KINDS}
        case["p0.01_over_ln"] = statistics.median(times["droq_p0.01"]) / statistics.median(times["ln"])
        case["launches"] = {k: handles[k][0].launches_per_step for k in KINDS}
        for kind in ("ln", "droq_p0.01"):
            core, ring = handles[kind]
            prof = core.profile_step(ring, iters=50)
            ln = [(label, ms * 1e3) for label, ms in prof if label.startswith("ln_")]
            case[f"{kind}_launch_us"] = dict(ln)
            case[f"{kind}_ln_sum_us"] = sum(us for _, us in ln)
            case[f"{kind}_step_sum_us"] = sum(ms for _, ms in prof) * 1e3
        case["step_ms"] = times
        res["cases"][name] = case
        print(json.dumps({name: case}), flush=True)
        for core, ring in handles.values():
            ring.close()
            core.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[droq_bench] {time.time() - t0:.0f} s", file=sys.stderr)
