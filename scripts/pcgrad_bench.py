"""PCGrad and CAGrad: cost of the pcgrad plan against the default plan, and the in-graph times of its new launches.

  python scripts/pcgrad_bench.py [--steps 1000] [--warmup 100] [--legs MS_x1,MS_x10,C10M_x1,C10O_x1] [--out FILE]

Workloads, each on a 128 Ki-transition device ring:
  MS_x1, MS_x10   the MT10 MTSAC shape (39 + 10 one-hot inputs, 4 actions, 400-wide 3-layer networks, batch 1280, 10 tasks,
                  precision 1, per-layer plan), 1 learner and 10 learners in one handle;
  C10M_x1, C10O_x1  the MT10 CARE shape of the same MLPs (BASELINE config 5: K = 6 mixture encoders 39 -> 50 -> 50, 768-d
                  task embedding, 50-wide context net), CARE(M) and CARE(O), 1 learner.
Each leg alternates four handles three times and reports the median: no pcgrad, pcgrad with both switches off (the Gram
matrix only), pcgrad on, and CAGrad (both PCGrad switches off, c = 0.5 on both optimizers).  The timeline run gives the
in-graph times of the pcgrad launches and, on the CARE legs, of care_tab_wgrad and the mixture-encoder weight-gradient
launches (the gemm launches between care_mix_bwd and care_tab_reduce).  The card's name, power limit and SM clock are read
in the same run (nvidia-smi, read-only query).
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

MODES = ("default", "switch_off", "on", "cagrad")
CAGRAD_C = 0.5


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power, clock = [x.strip() for x in q.split(",")]
        return {"name": name, "power_limit": power, "max_sm_clock": clock}
    except Exception as e:                     # noqa: BLE001 -- reported, not fatal
        return {"error": repr(e)}


def config(R, pcgrad, care=None):
    """care: None (MTSAC), "M" or "O" (the CARE variant)."""
    from distributed_sac_b200.core import CoreConfig
    kw = {}
    if care:
        kw = dict(care=True, num_encoders=6, mix_hidden=[50], mix_out=50, ctx_in=768, ctx_hidden=[50, 50], ctx_out=50,
                  tau_se=0.05, care_original=care == "O", emb_dim=50, lr_ctx=3e-4)
    return CoreConfig(state_dim=39, act_dim=4, actor_hidden=[400] * 3, critic_hidden=[400] * 3, batch=1280, num_tasks=10,
                      weighted_loss=care != "O", replicas=R, precision=1, pcgrad=pcgrad, **kw)


def _timed(names):
    """Indices of the launches a timeline reports: the surgery's, the Adam launches after them and the CARE weight
    gradients (care_tab_wgrad, and the mixture-encoder launches between care_mix_bwd and care_tab_reduce)."""
    lo, hi = (names.index("care_mix_bwd"), names.index("care_tab_reduce")) if "care_mix_bwd" in names else (0, 0)
    return [i for i, n in enumerate(names) if n.startswith("pcgrad") or lo < i < hi or
            n in ("adam_critic+polyak", "adam_actor+alpha", "care_tab_wgrad")]


def leg(R, ring_n, steps, warmup, mode, timeline, care=None):
    import torch
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(config(R, mode != "default", care), 0, seed=11)
    ring = Replay(core, ring_n, seed=3)
    ring.fill_synthetic(ring_n, seed=5)
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        if mode in ("switch_off", "cagrad"):
            core.set_pcgrad(critic=False, actor=False)
        if mode == "cagrad":
            core.set_cagrad(critic=CAGRAD_C, actor=CAGRAD_C)
        core.prepare(ring)
        core.step_sampled(ring, warmup)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        core.step_sampled(ring, steps)
        e1.record()
    e1.synchronize()
    us = 1e3 * e0.elapsed_time(e1) / steps
    assert torch.isfinite(core.read_losses(64)[:, :, 0]).all()
    extra = {}
    if mode != "default":
        rec = core.read_pcgrad(0)
        extra = {"critic_projections": int(rec["projected"][0].sum()), "actor_projections": int(rec["projected"][1].sum())}
        if mode == "cagrad":
            cg = core.read_cagrad(0)
            extra = {"ibest": cg["ibest"].tolist(), "lambda": cg["lambda"].tolist(), "w": rec["w"].tolist()}
    tl = None
    if timeline:
        with torch.cuda.stream(stream):
            names = ["sample", "ingest"] + [n for n, _ in core.profile_step(ring, iters=2)][1:]
            t = core.graph_timeline(ring, iters=200)
        torch.cuda.synchronize()
        tl = {"new_launches_us": {f"{i}:{names[i]}": t[i] for i in _timed(names)},
              "launches": len(names), "step_us": sum(t), "all_us": dict(zip(names, t))}
    ring.close()
    core.close()
    return us, tl, extra


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=1000)
    ap.add_argument("--warmup", type=int, default=100)
    ap.add_argument("--legs", default="MS_x1,MS_x10,C10M_x1,C10O_x1")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    import __graft_entry__ as ge
    ge.build()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("pcgrad_bench.py needs a CUDA device")
    res = {"card": card(), "steps": args.steps, "warmup": args.warmup, "legs": {}}
    legs = (("MS_x1", 1, 1 << 17, None), ("MS_x10", 10, 1 << 17, None), ("C10M_x1", 1, 1 << 17, "M"),
            ("C10O_x1", 1, 1 << 17, "O"))
    for name, R, ring_n, care in legs:
        if name not in args.legs.split(","):
            continue
        us = {m: [] for m in MODES}
        tls, extras = {}, {}
        for k in range(3):
            for m in MODES:
                t, tl, ex = leg(R, ring_n, args.steps, args.warmup, m, timeline=(k == 0 and R == 1), care=care)
                us[m].append(t)
                extras[m] = ex
                if tl is not None:
                    tls[m] = tl
        med = {m: statistics.median(v) for m, v in us.items()}
        out = {"learners": R, "ring_per_learner": ring_n, "us_per_step": med,
               "switch_off_over_default": med["switch_off"] / med["default"], "on_over_default": med["on"] / med["default"],
               "cagrad_over_default": med["cagrad"] / med["default"], "cagrad_over_on": med["cagrad"] / med["on"],
               "last_step_projections": extras, "runs_us": us}
        if tls:                        # start-to-start times of the unforked timeline run (b200sac_graph_timeline)
            out["graph_timeline"] = tls
            out["pcgrad_launches_us"] = {m: {k: v for k, v in tl["new_launches_us"].items() if "pcgrad" in k}
                                         for m, tl in tls.items()}
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
    print(f"[pcgrad_bench] {time.time() - t0:.0f} s", file=sys.stderr)
