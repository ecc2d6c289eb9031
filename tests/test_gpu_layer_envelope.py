"""The per-layer step plan (build_plan_layered in b200sac.cu, plain SAC / MTSAC outside the layer-chained envelope) at both precisions,
against the autograd oracle.

The per-layer plan carries every precision = 1 learner, the 400-wide VS / MS shapes, the many-learner configurations and
every exact-fp32 learner outside the chained envelope.  Per launch group the plan builder picks an engine (wgmma 3xTF32,
32x32 FFMA, or the thin input-layer kernel), a wgmma tile width (64 / 128 / 160) and a split-K factor (4 / 2 / 1); the head
backward takes the 8-column or the 128-bit kernel, with or without row slices; large batches compute the policy-head output
gradient in a kernel of its own.  The cases (_harness.LAYER_CASES) reach each of those choices (test_sweep_covers_every_branch names any
that a change of the table stops reaching), at the shapes where kernels go wrong: batch 1 and 2048, odd pitches, K tails of
split weight gradients, padded first layers, 1 and 8 hidden layers, act_dim 1 and 8, 33 and 64 tasks.  Every step is checked
with the CUDA step's ReLU masks forced into the oracle (tests/_golden.py::kink_checked_step): losses, every parameter /
target / Adam moment, and every per-row output element by element.  Guards keep the sweep from passing vacuously: the plan's
launch labels read back from the handle equal the mirror's below, every hidden layer is partly active, every trainable
tensor moves, and the pad columns of padded first layers stay exactly zero.
"""
from collections import namedtuple

import pytest
import torch

import sac_port as sp
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, kink_checked_step, sync_core_to_port
from _harness import (LAYER_CASES, REPLICA_SPEC, REPLICAS, _eps, _pad4, _params, _sms, chained_launches, check_active,
                      check_losses, check_rows, cuda, plan_labels, run_checked)

gpu = pytest.mark.gpu

# A VS-like learner at precision 1 (batch >= 512 and not a multiple of 128) run with each wgmma tile forced:
# id -> (B200SAC_TC_BN, B200SAC_TC_PAIR128)
TILE_SPEC = dict(state_dim=39, num_tasks=0, act_dim=4, actor_hidden=[400, 400], critic_hidden=[400, 400], batch=1000)
TILES = {"128x64": ("64", "0"), "128x128": ("128", "0"), "128x128-paired": ("128", "1"), "128x160": ("160", "0")}

H100_SMS = 132


# ---------------------------------------------------------------------------------------------------------------------
# mirror of the per-layer plan builder (build_plan_layered / gemm_launch / head_bwd in b200sac.cu)
# ---------------------------------------------------------------------------------------------------------------------
FWD, DGRAD, WGRAD = "fwd", "dgrad", "wgrad"
SPLIT_K, SPLIT_K_MIN = 4, 512          # kSplitK, kSplitKMin
TC_BM, TC_BK = 128, 32
GT_NMAX, GT_KC = 16, 512               # gemm_thin.cuh: widest thin N, K rows per pass

# one GEMM problem: the pitches of its A / B operands (every base address is 16-B aligned when its pitch is a multiple of
# 4 floats: second-network offsets net * B * in, the s half of [s'; s] at B * ld, K slices at multiples of 32 rows); `inp`:
# a problem of a first (input) layer
Prob = namedtuple("Prob", "mode M N K lda ldb inp")
# one plan launch: label, engine ("wgmma" | "ffma" | "thin" | None), tile width, split factor, the problems it runs and
# whether its group also issued a launch on the other engine
Launch = namedtuple("Launch", "label engine bn split probs mixed")


def tc_eligible(p):
    return p.lda % 4 == 0 and p.ldb % 4 == 0 and p.M >= 32 and p.N >= 32 and p.K >= 32


def gemm_is_thin(p):
    return p.mode != FWD and p.N <= GT_NMAX


def tc_group_cost(v, bn, R, sms, pair128=False):
    tiles = sum(-(-p.M // TC_BM) * -(-p.N // bn) for p in v)
    nk = max([1] + [-(-p.K // TC_BK) for p in v])
    chunk = 3100.0 if (bn == 128 and pair128) else 1200.0 + 11.7 * bn
    tile = 3000.0 + nk * chunk + 38.0 * bn
    return float(-(-(tiles * R) // sms)) * tile


def tc_pick_bn(v, R, sms, force_bn=None, pair128=False):
    if force_bn is not None:
        return force_bn
    max_n = max(p.N for p in v)
    best, cost = 64, tc_group_cost(v, 64, R, sms, pair128)
    for bn in (128, 160):
        if max_n < 2 * bn - 64:
            continue
        c = tc_group_cost(v, bn, R, sms, pair128)
        if c < cost:
            best, cost = bn, c
    return best


def _splits(p, S, gslices):
    """expand: the K slices of one problem (weight gradients with K >= 512, 32-row multiples but the last)."""
    if not (p.mode == WGRAD and p.K >= SPLIT_K_MIN and gslices > 1) or S == 1:
        return [p]
    ln = (-(-p.K // S) + 31) & ~31
    return [p._replace(K=min(ln, p.K - kb)) for kb in range(0, p.K, ln)]


def _gemm_label(probs, engine, bn, pair, split):
    p0, pl = probs[0], probs[-1]
    kind = {FWD: "gemm_fwd", DGRAD: "gemm_dgrad"}.get(p0.mode) or (
        "gemm_wgrad+dgrad" if pl.mode == DGRAD and engine != "thin" else "gemm_wgrad")   # thin: named after p0 alone
    what = f"wgmma 128x{bn}{' paired' if pair else ''}" if engine == "wgmma" else engine
    return f"{kind}({what}{f', split {split}' if any(p.mode == WGRAD for p in probs) else ''})"


def gemm_launch(ps_in, precision, gslices, R, sms, force_bn=None, pair128=False):
    """The launches of one GEMM group: split factor (precision 1: the cheapest under tc_group_cost; FFMA: the finest),
    then a wgmma launch for the eligible problems and an FFMA / thin launch for the rest."""
    expand = lambda S: [q for p in ps_in for q in _splits(p, S, gslices)]
    S = SPLIT_K
    if precision == 1:
        best = float("inf")
        for s in (4, 2, 1):
            o = [p for p in expand(s) if tc_eligible(p)]
            if not o:
                S = s
                break
            cost = tc_group_cost(o, tc_pick_bn(o, R, sms, force_bn, pair128), R, sms, pair128)
            if cost < best:
                best, S = cost, s
    ps = expand(S)
    split = S if any(p.mode == WGRAD and p.K >= SPLIT_K_MIN for p in ps_in) and gslices > 1 else 1
    out = []
    if precision == 1:
        tc, rest = [p for p in ps if tc_eligible(p)], [p for p in ps if not tc_eligible(p)]
        if tc:
            bn = tc_pick_bn(tc, R, sms, force_bn, pair128)
            pair = bn == 128 and pair128
            out.append(Launch(_gemm_label(tc, "wgmma", bn, pair, split), "wgmma", bn, split, tc, bool(rest)))
        ps = rest
    if ps:
        engine = "thin" if all(gemm_is_thin(p) for p in ps) else "ffma"
        out.append(Launch(_gemm_label(ps, engine, 0, False, split), engine, 0, split, ps, bool(out)))
    return out


def _net(in0, hidden, out):
    """(in, out, ld) per layer; first layers have 16-B row pitches"""
    dims = [in0] + list(hidden) + [out]
    return [(i, o, _pad4(i) if l == 0 else i) for l, (i, o) in enumerate(zip(dims[:-1], dims[1:]))]


def head_bwd_label(policy, width, gslices):
    wide = not policy and width % 4 == 0
    return f"head_bwd({'policy' if policy else 'q'}, {'128-bit, ' if wide else ''}row slices {gslices})"


def mirror_plan(spec, precision, R=1, sms=H100_SMS, force_bn=None, pair128=False):
    """[Launch] of the per-layer plan, in plan order, with the labels b200sac_profile_step gives them ("sample+ingest"
    first)."""
    B, A = spec.batch, spec.act_dim
    obs = spec.state_dim + spec.num_tasks
    actor, critic = _net(obs, spec.actor_hidden, 2 * A), _net(obs + A, spec.critic_hidden, 1)
    La, Lc = len(spec.actor_hidden), len(spec.critic_hidden)
    gslices = SPLIT_K if B >= SPLIT_K_MIN else 1
    use_fork = precision == 0
    plan = [Launch("sample+ingest", None, 0, 1, [], False)]
    fwd = lambda M, lo, l: Prob(FWD, M, lo[1], lo[0], lo[2], lo[2], l == 0)
    wgrad = lambda lo, l: Prob(WGRAD, lo[1], lo[0], B, lo[1], lo[2], l == 0)
    dgrad = lambda lo, l: Prob(DGRAD, B, lo[0], lo[1], lo[1], lo[2], l == 0)
    launch = lambda ps: plan.extend(gemm_launch(ps, precision, gslices, R, sms, force_bn, pair128))
    other = lambda label: plan.append(Launch(label, None, 0, 1, [], False))
    for l in range(max(La, Lc)):                                  # A: actor on [s'; s], Q1, Q2 on (s, a)
        ps = ([fwd(2 * B, actor[l], l)] if l < La else []) + ([fwd(B, critic[l], l)] * 2 if l < Lc else [])
        if use_fork and La == Lc:
            launch(ps[1:])
            launch(ps[:1])
        else:
            launch(ps)
    other("policy_head")
    for l in range(Lc):                                           # B: target critics on (s', a')
        launch([fwd(B, critic[l], l)] * 2)
    other("critic_heads")
    other(head_bwd_label(False, spec.critic_hidden[-1], gslices))
    for l in reversed(range(Lc)):                                 # C: critic backward
        ps = [wgrad(critic[l], l)] * 2 + ([dgrad(critic[l], l)] * 2 if l > 0 else [])
        if use_fork and l > 0:
            launch(ps[:2])
            launch(ps[2:])
        else:
            launch(ps)
    other("adam_critic+polyak")
    for l in range(Lc):                                           # D: the updated critics on (s, a~)
        launch([fwd(B, critic[l], l)] * 2)
    other("actor_q_heads")
    other(head_bwd_label(False, spec.critic_hidden[-1], gslices))
    for l in reversed(range(Lc)):
        launch([dgrad(critic[l], l)] * 2)
    if B * A > 2048:                                              # E: policy backward
        other("policy_dout")
    other(head_bwd_label(True, spec.actor_hidden[-1], gslices))
    for l in reversed(range(La)):
        ps = [wgrad(actor[l], l)] + ([dgrad(actor[l], l)] if l > 0 else [])
        if use_fork and l > 0:
            launch(ps[:1])
            launch(ps[1:])
        else:
            launch(ps)
    other("adam_actor+alpha")
    return plan


def chained(spec, precision):
    """fused_eligible: the layer-chained plan takes the learner."""
    widths = list(spec.actor_hidden) + list(spec.critic_hidden)
    return (precision == 0 and all(w % 4 == 0 and w <= 256 for w in widths)
            and spec.state_dim + spec.num_tasks + spec.act_dim <= 252)


def padded(spec):
    obs = spec.state_dim + spec.num_tasks
    return obs % 4 != 0 or (obs + spec.act_dim) % 4 != 0


def features(spec, precision, R=1, sms=H100_SMS, force_bn=None, pair128=False):
    """The branches of the plan and its kernels that one handle reaches, by name."""
    plan = mirror_plan(spec, precision, R, sms, force_bn, pair128)
    B, A = spec.batch, spec.act_dim
    have = set()
    for ln in plan:
        if ln.engine is None:
            if ln.label.startswith("head_bwd(q"):
                have.add(f"head_bwd {'128-bit' if '128-bit' in ln.label else 'narrow'}, "
                         f"{'row slices' if B >= SPLIT_K_MIN else 'no slices'}")
            continue
        if ln.engine == "wgmma" and force_bn is None:
            have.add(f"cost model: tile 128x{ln.bn}")
            if B >= SPLIT_K_MIN and any(p.mode == WGRAD for p in ln.probs):
                have.add(f"cost model: split {ln.split}")
        if ln.mixed:
            have.add("mixed wgmma + FFMA group")
        if any(p.inp for p in ln.probs):
            have.add(f"input layer: {ln.engine}")
        if ln.split > 1:
            if any(p.mode == WGRAD and p.K % 8 for p in ln.probs):
                have.add("K-tail slice")
            if ln.engine == "thin":
                have.add("thin on K slices")
        if ln.engine == "thin" and any(p.K > GT_KC for p in ln.probs):
            have.add("thin: several K passes")
    if B * A > 2048:
        have.add(f"policy_dout, {'row slices' if B >= SPLIT_K_MIN else 'no slices'}")
    if B in (1, 2048):
        have.add(f"batch {B}")
    for n in (len(spec.actor_hidden), len(spec.critic_hidden)):
        if n in (1, 8):
            have.add(f"{n} hidden layers")
    if A in (1, 8):
        have.add(f"act_dim {A}")
    if spec.num_tasks in (33, 64):
        have.add(f"{spec.num_tasks} tasks")
    if padded(spec):
        have.add("padded first layer")
    return have


WANT = {"cost model: tile 128x64", "cost model: tile 128x128", "cost model: tile 128x160",
        "cost model: split 4", "cost model: split 2", "cost model: split 1",
        "head_bwd narrow, no slices", "head_bwd narrow, row slices", "head_bwd 128-bit, no slices",
        "head_bwd 128-bit, row slices", "policy_dout, no slices", "policy_dout, row slices",
        "input layer: thin", "input layer: ffma", "input layer: wgmma", "mixed wgmma + FFMA group",
        "batch 1", "batch 2048", "K-tail slice", "thin on K slices", "thin: several K passes", "1 hidden layers", "8 hidden layers",
        "act_dim 1", "act_dim 8", "64 tasks", "33 tasks", "padded first layer"}


# ---------------------------------------------------------------------------------------------------------------------
# CPU: the sweep reaches every branch; the mirror agrees with shapes worked out by hand
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", list(LAYER_CASES))
def test_case_is_outside_the_chained_envelope(name):
    assert not chained(sp.SacSpec(**LAYER_CASES[name]), 0), name


def test_sweep_covers_every_branch():
    have = set()
    for c in LAYER_CASES.values():
        for precision in (0, 1):
            have |= features(sp.SacSpec(**c), precision)
    have |= features(sp.SacSpec(**REPLICA_SPEC), 1, R=REPLICAS)
    missing = sorted(WANT - have)
    assert not missing, f"on {H100_SMS} SMs no case reaches: {missing}"


def test_replica_shape_changes_the_tensor_core_choices():
    spec = sp.SacSpec(**REPLICA_SPEC)
    assert not chained(spec, 0) and spec.batch % spec.num_tasks == 0
    l1 = [ln.label for ln in mirror_plan(spec, 1, R=1)]
    l3 = [ln.label for ln in mirror_plan(spec, 1, R=REPLICAS)]
    assert l1 != l3 and len(l1) == len(l3)


def test_mirror_matches_hand_worked_shapes():
    s517 = sp.SacSpec(**LAYER_CASES["split517"])
    assert [p.K for p in _splits(Prob(WGRAD, 96, 10, 517, 96, 12, True), 4, 4)] == [160, 160, 160, 37]
    rows_per = -(-517 // 4)
    assert [min(rows_per, 517 - r0) for r0 in range(0, 517, rows_per)] == [130, 130, 130, 127]
    thin = [ln for ln in mirror_plan(s517, 0) if ln.engine == "thin"]
    assert thin and all(ln.split == 4 for ln in thin if any(p.mode == WGRAD for p in ln.probs))
    assert "policy_dout" in [ln.label for ln in mirror_plan(sp.SacSpec(**LAYER_CASES["pdout257"]), 0)]
    assert "policy_dout" not in [ln.label for ln in mirror_plan(sp.SacSpec(**LAYER_CASES["pdout256"]), 0)]
    # DESIGN.md 4.2: 29 launches per step for the 3-hidden-layer VS shape at precision 1, index sampling included
    vs = sp.vs_spec()
    assert len(mirror_plan(vs, 1)) + 1 == 29
    assert all(ln.engine == "wgmma" for ln in mirror_plan(vs, 1) if ln.engine and not any(p.inp for p in ln.probs))
    b1 = mirror_plan(sp.SacSpec(**LAYER_CASES["b1"]), 1)
    assert all(ln.engine in (None, "ffma", "thin") for ln in b1)


# ---------------------------------------------------------------------------------------------------------------------
# helpers of the GPU tests
# ---------------------------------------------------------------------------------------------------------------------
def check_plan(spec, precision, what, R=1, env=None):
    """A throwaway handle created under `env` runs the per-layer plan the mirror predicts.  The labels are read with the
    environment restored: the handle keeps what it chose when it was built."""
    from distributed_sac_b200.core import SacCore
    with pytest.MonkeyPatch.context() as mp:
        for k, v in (env or {}).items():
            mp.setenv(k, v)
        core = SacCore(core_config(spec, replicas=R, precision=precision), 0, seed=0)
    force_bn = int(env["B200SAC_TC_BN"]) if env else None
    pair = bool(env) and env.get("B200SAC_TC_PAIR128") == "1"
    want = [ln.label for ln in mirror_plan(spec, precision, R, _sms(), force_bn, pair)]
    got = plan_labels(core)
    core.close()
    assert got == want, f"{what}: plan labels differ from the mirror's:\n got  {got}\n want {want}"
    return want


def check_pad_columns(core, spec, what):
    """Pad columns of the padded first layers (weights, targets, gradients, both Adam moments) are exactly zero."""
    from distributed_sac_b200 import _lib
    n = 0
    for which, arena in (("params", _lib.PARAMS), ("grads", _lib.GRADS), ("adam_m", _lib.ADAM_M), ("adam_v", _lib.ADAM_V)):
        flat = core.export_arena(arena)
        for name, (off, rows, cols, trainable, _opt, pitch) in core.table.items():
            if pitch == cols or (arena != _lib.PARAMS and not trainable):
                continue
            pad = flat[off:off + rows * pitch].reshape(rows, pitch)[:, cols:]
            assert not pad.any(), f"{what}: {which} {name} has non-zero pad columns: {pad[pad != 0][:8].tolist()}"
            n += 1
    assert n >= 4, f"{what}: only {n} padded tensors"     # actor.0 or q1/q2(.target).0 weights in all four arenas


def check_moved(core, spec, p, what):
    from distributed_sac_b200 import _lib
    got = core.get_named(_lib.PARAMS)
    for k in sp.param_names(spec, sp.TRAINABLE_NETS):
        assert torch.isfinite(got[k]).all(), (what, k)
        assert not torch.equal(got[k], p[k]), f"{what}: {k} did not change"


def run_case(spec, precision, what, chained_launches, env=None, n_steps=2):
    from distributed_sac_b200.core import SacCore
    check_plan(spec, precision, what, env=env)
    p = _params(spec, seed=7)
    port = sp.PortLearner(spec, p)
    with pytest.MonkeyPatch.context() as mp:
        for k, v in (env or {}).items():
            mp.setenv(k, v)
        core = SacCore(core_config(spec, precision=precision), 0, seed=0)
        assert core.launches_per_step != chained_launches, what
        assert core.launches_per_step == len(mirror_plan(spec, precision)), what
        flips, worst = run_checked(core, spec, port, n_steps, seed=13, what=what)
        check_moved(core, spec, p, what)
        if padded(spec):
            check_pad_columns(core, spec, what)
        core.close()
    print(f"[kinks] {what}: {flips} mask bits differed, all at numerically-zero pre-activations")
    print(f"[rows] {what}: largest per-row |got - ref| / (|ref| + mean|ref|) = {worst:.2e}")


# ---------------------------------------------------------------------------------------------------------------------
# 1: the oracle sweep at both precisions
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("name", list(LAYER_CASES))
def test_per_layer_step_matches_oracle(cuda, chained_launches, name, precision):
    run_case(sp.SacSpec(**LAYER_CASES[name]), precision, f"{name} precision {precision}", chained_launches)


# ---------------------------------------------------------------------------------------------------------------------
# 2: every wgmma tile inside a full step
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("tile", list(TILES))
def test_forced_tile_step_matches_oracle(cuda, chained_launches, tile):
    bn, pair = TILES[tile]
    env = {"B200SAC_TC_BN": bn, "B200SAC_TC_PAIR128": pair}
    spec = sp.SacSpec(**TILE_SPEC)
    labels = [ln.label for ln in mirror_plan(spec, 1, force_bn=int(bn), pair128=pair == "1")]
    assert sum(f"wgmma {tile.replace('-', ' ')}" in n for n in labels) >= 8, labels
    run_case(spec, 1, f"tile {tile}", chained_launches, env=env)


# ---------------------------------------------------------------------------------------------------------------------
# 3: co-scheduled replicas with parameters, minibatches and task ids of their own
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
def test_replicas_with_different_parameters_match_their_oracles(cuda, chained_launches, precision):
    """Each replica follows its own oracle; at precision 0 each also equals bit for bit an R = 1 handle given the same
    state and inputs (fixed splits); at precision 1 the R = 3 handle runs other tiles / split factors than an R = 1 one,
    and the R = 1 handle given each replica's state and inputs follows the oracle as well."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    spec, R = sp.SacSpec(**REPLICA_SPEC), REPLICAS
    want = check_plan(spec, precision, f"R = {R}", R=R)
    if precision == 1:
        assert want != check_plan(spec, precision, "R = 1")
    params = [_params(spec, seed=30 + r) for r in range(R)]
    ports = [sp.PortLearner(spec, p) for p in params]
    batches = [sp.synthetic_batch(spec, seed=300 + r) for r in range(R)]
    gen = torch.Generator().manual_seed(3)
    eps = [_eps(spec, gen) for _ in range(R)]
    tids = [torch.argmax(b[0][:, -spec.num_tasks:], dim=1) for b in batches]
    assert not torch.equal(tids[0], tids[1]) and not torch.equal(tids[1], tids[2])

    core = SacCore(core_config(spec, replicas=R, precision=precision), 0, seed=0)
    assert core.launches_per_step != chained_launches
    for r in range(R):
        sync_core_to_port(core, ports[r], r)
    core.step(*[torch.stack([b[j] for b in batches]) for j in range(5)],
              torch.stack([e[0] for e in eps]), torch.stack([e[1] for e in eps]))
    for r in range(R):
        forced = cuda_relu_masks(core, spec, r)
        with sp.ReluTape(forced) as tape:
            o = ports[r].update_SAC(*batches[r], *eps[r], want_intermediates=True)
        check_forced(tape, forced, f"replica {r}: ")
        check_active(core, spec, r, f"replica {r}: ")
        check_losses(core, o, r, f"replica {r}: ")
        check_port_state(core, ports[r], replica=r)
        check_rows(core, spec, o, r, f"replica {r}: ")
    L3 = core.read_losses(1)[0]
    assert not torch.equal(L3[0], L3[1]) and not torch.equal(L3[1], L3[2])

    if precision == 0:
        single = SacCore(core_config(spec, precision=0), 0, seed=0)
        for r in range(R):
            sync_core_to_port(single, sp.PortLearner(spec, params[r]))
            single.step(*batches[r], *eps[r])
            diff = [f"{which}:{k}" for which, arena in (("params", _lib.PARAMS), ("grads", _lib.GRADS), ("adam_m", _lib.ADAM_M),
                                                         ("adam_v", _lib.ADAM_V))
                    for a, b in [(core.get_named(arena, r), single.get_named(arena))] for k in a if not torch.equal(a[k], b[k])]
            assert not diff, f"replica {r} of the R = 3 handle differs from the R = 1 handle in {diff[:8]}"
            assert torch.equal(L3[r], single.read_losses(1)[0, 0]), (r, L3[r].tolist(), single.read_losses(1)[0, 0].tolist())
        single.close()
    else:
        # the R = 1 handle's own tiles and split factors, on each replica's state and inputs, against the oracle too
        single = SacCore(core_config(spec, precision=1), 0, seed=0)
        for r in range(R):
            port = sp.PortLearner(spec, params[r])
            o, _ = kink_checked_step(single, port, spec, batches[r], *eps[r], want_intermediates=True)
            what = f"R = 1 handle, replica {r}'s inputs: "
            check_active(single, spec, 0, what)
            check_losses(single, o, 0, what)
            check_port_state(single, port)
            check_rows(single, spec, o, 0, what)
        single.close()
    core.close()
