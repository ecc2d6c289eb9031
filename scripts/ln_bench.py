"""Layer-normalized critics (b200sac_cfg.critic_ln): what the LayerNorm launches cost a sampled step.

  python scripts/ln_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Leg 1: steps/s of sampled steps from a 1 Mi-transition device ring at the bench.py shapes LL (precision 0; one replica and
16 replicas), VS and MS (precision 1, one replica), for three handles of each: the per-layer plan without LayerNorm
(B200SAC_FUSE=0 at LL, where the layer-chained plan is the default), the per-layer plan with critic_ln, and the default
plan (the layer-chained one at LL).  The handles alternate three times and the median is reported.  Leg 2: the device
time of every LayerNorm launch of one step (b200sac_profile_step, CUDA events around each launch of an eager step) and
their sum beside the whole step's.  The card's name, power limit and maximum SM clock are read in the same run
(nvidia-smi, read-only).
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
KINDS = ("per_layer", "per_layer_ln", "default")


def make(workload, R, precision, kind):
    from bench import core_config
    from distributed_sac_b200.core import SacCore
    cfg = core_config(workload, R, precision=precision)
    cfg.critic_layer_norm = kind == "per_layer_ln"
    old = os.environ.pop("B200SAC_FUSE", None)
    if kind == "per_layer":
        os.environ["B200SAC_FUSE"] = "0"
    try:
        return SacCore(cfg, 0, seed=11)
    finally:
        os.environ.pop("B200SAC_FUSE", None)
        if old is not None:
            os.environ["B200SAC_FUSE"] = old


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
        raise SystemExit("ln_bench.py needs a CUDA device")
    from distributed_sac_b200.core import Replay
    res = {"card": card(), "steps": args.steps, "cases": {}}
    for workload, R, precision in CASES:
        name = f"{workload} R={R} precision {precision}"
        handles = {}
        for kind in KINDS:
            core = make(workload, R, precision, kind)
            ring = Replay(core, 1 << 20, "device", seed=3)
            ring.fill_synthetic(1 << 20, seed=5)
            core.prepare(ring)
            handles[kind] = (core, ring)
        times = {k: [] for k in KINDS}
        for _ in range(3):
            for kind in KINDS:
                times[kind].append(run_ms(*handles[kind], args.steps, args.warmup))
        core, ring = handles["per_layer_ln"]
        prof = core.profile_step(ring, iters=50)
        ln = [(label, ms * 1e3) for label, ms in prof if label.startswith("ln_")]
        case = {f"{k}_steps_per_s": 1e3 / statistics.median(times[k]) for k in KINDS}
        case.update(ln_over_per_layer=statistics.median(times["per_layer_ln"]) / statistics.median(times["per_layer"]),
                    launches={k: handles[k][0].launches_per_step for k in KINDS},
                    ln_launch_us=dict(ln), ln_sum_us=sum(us for _, us in ln),
                    step_sum_us=sum(ms for _, ms in prof) * 1e3, step_ms=times)
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
    print(f"[ln_bench] {time.time() - t0:.0f} s", file=sys.stderr)
