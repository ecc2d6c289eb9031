"""Critic ensembles (b200sac_cfg.critic_ensemble): what E critics cost a sampled step.

  python scripts/ensemble_bench.py [--steps 2000] [--warmup 200] [--out FILE]

Steps/s of sampled steps (graph launches from a 1 Mi-transition device ring) at the bench.py shapes LL (precision 0) and
VS (precision 1), one replica, for: the twin per-layer plan (critic_ensemble = 0, B200SAC_FUSE=0 so that LL runs the
per-layer plan too), E = 2, 5 and 10 with m = 2 and the mean actor reduction, and RLPD's leg: E = 10, m = 2, LayerNorm
critics and a prior-data ring at fraction 0.5.  The legs alternate five times and the median is reported.  The card's
name, power limit and maximum SM clock are read in the same run (nvidia-smi, read-only).
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

CASES = [("LL", 0), ("VS", 1)]
LEGS = {"twin": dict(E=0), "E2": dict(E=2), "E5": dict(E=5), "E10": dict(E=10), "rlpd": dict(E=10, ln=True, prior=0.5)}
RING = 1 << 20


def make(workload, precision, E, ln=False, prior=None):
    from bench import core_config
    from distributed_sac_b200.core import Replay, SacCore
    cfg = core_config(workload, 1, precision=precision)
    cfg.critic_ensemble = E
    cfg.critic_layer_norm = ln
    os.environ["B200SAC_FUSE"] = "0"
    try:
        core = SacCore(cfg, 0, seed=11)
    finally:
        del os.environ["B200SAC_FUSE"]
    if E:
        core.set_ensemble(2, "mean")
    ring = Replay(core, RING, "device", seed=3)
    ring.fill_synthetic(RING, seed=5)
    keep = [ring]
    if prior is not None:
        pr = Replay(core, RING, "device", seed=4)
        pr.fill_synthetic(RING, seed=6)
        ring.attach_prior(pr)
        ring.set_prior_rows(int(prior * cfg.batch + 0.5))
        keep.append(pr)
    core.prepare(ring)
    return core, ring, keep


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
        raise SystemExit("ensemble_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "cases": {}}
    for workload, precision in CASES:
        name = f"{workload} precision {precision}"
        handles = {leg: make(workload, precision, **kw) for leg, kw in LEGS.items()}
        times = {leg: [] for leg in LEGS}
        for _ in range(5):
            for leg, (core, ring, _) in handles.items():
                times[leg].append(run_ms(core, ring, args.steps, args.warmup))
        case = {f"{leg}_us_per_step": 1e3 * statistics.median(t) for leg, t in times.items()}
        case.update({f"{leg}_over_twin": statistics.median(t) / statistics.median(times["twin"]) for leg, t in times.items()})
        case["launches"] = {leg: h[0].launches_per_step for leg, h in handles.items()}
        case["step_ms"] = times
        res["cases"][name] = case
        print(json.dumps({name: case}), flush=True)
        for core, ring, keep in handles.values():
            for rb in keep:
                rb.close()
            core.close()
    line = json.dumps(res)
    print(line)
    if args.out:
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    t0 = time.time()
    main()
    print(f"[ensemble_bench] {time.time() - t0:.0f} s", file=sys.stderr)
