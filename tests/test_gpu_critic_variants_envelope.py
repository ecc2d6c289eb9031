"""The three critic variants of the per-layer step -- LayerNorm critics (critic_ln), dropout Q-functions (critic_dropout,
DroQ) and critic ensembles (critic_ensemble, REDQ / RLPD) -- over the per-layer plan's envelope at both precisions, against
the autograd oracles (oracle/critic_ln_port.py, oracle/droq_port.py, oracle/redq_port.py).

The variants' own kernels (ln_kernels.cuh; the E-critic head, head-backward and policy-dout kernels of sac_kernels.cuh)
go wrong where their loops and index arithmetic change shape: a partial last ln_bwd chunk (batch not a
multiple of kLnRows = 16) and 128 chunks through its ticket (batch 2048), a second pass of ln_bwd's column loop (H > 256),
drop_row's group loop past its first 32 groups (H > 128) and odd widths, split-K weight gradients and row-sliced head
gradients (batch >= 512, critic k's slots at + k * rsNet), head_bwd_kernel in critic mode (last width not a multiple of
4), policy_dout_kernel's E-sum (batch * act > 2048), a grouped GEMM cut into several launches (E = 10 at batch >= 512),
and the actor's "min" routing over E critics.  CASES reaches each of these (test_cases_reach_every_edge fails if an edit of
the table stops reaching one):

  1  step parity, both precisions: five steps from an oracle state synced into the handle, the device's ReLU masks and
     actor routing forced into the oracle; every gradient Adam reads (LayerNorm dg / dc of every critic and layer
     included), every parameter, target and Adam moment, the losses and every per-row output (q_1 .. q_E included) within
     REL; the plan branch each case is there for, every critic tensor moving, a non-zero drop fraction, "min" routing to
     critics other than critic 1;
  2  the normalization launches alone: h == relu(LN(z)) in fp64 for every pass, layer, critic and replica;
  3  the dropout masks bit for bit against philox_ref.drop_masks(nets=E) over three steps, one of them critic-only;
  4  replica independence: replica r of an R = 3 handle equals an R = 1 handle bit for bit (precision 0);
  5  the edge coverage of the case table (CPU).
"""
import contextlib

import numpy as np
import pytest
import torch

import critic_ln_port as lnp
import droq_port as dq
import philox_ref as pr
import redq_port as rq
import sac_port as sp
from _golden import check_forced, check_port_state, core_config, cuda_relu_masks, sync_core_to_port
from _harness import (LAYER_CASES, REPLICA_SPEC, ROW_OUTPUTS, capture_grads, check_active, check_grads, check_losses,
                      check_rows, cuda, plan_labels)

gpu = pytest.mark.gpu
PARAMS, ADAM_M, ADAM_V, GRADS = 0, 1, 2, 3
SEED = 11
KINDS = {"Q": "cur", "T": "next", "P": "pi"}          # debug buffer letter -> pass
LN_ROWS, LN_THREADS, GS_MAXG, SPLIT_K_MIN = 16, 256, 24, 512     # kLnRows, kLnThreads, GS_MAXG, kSplitKMin

# id -> (SacSpec fields, variant, precisions).  variant: ln (LayerNorm), p (dropout rate, or one per replica: DroQ), E
# (critics; 2 = the twin handle), ens ((m, actor reduction), or one per replica), R (replicas).
RLPD = dict(state_dim=17, num_tasks=0, act_dim=6, actor_hidden=[256, 256], critic_hidden=[256, 256], batch=256)
VS1024 = dict(sp.vs_spec(batch=1024).to_json(), actor_hidden=[400, 400], critic_hidden=[400, 400])
CASES = {
    "ln-b1": (LAYER_CASES["b1"], dict(ln=True), (0, 1)),                    # batch 1, one hidden layer of 29
    "droq-b1": (LAYER_CASES["b1"], dict(ln=True, p=0.1), (0, 1)),
    "droq-odd67": (LAYER_CASES["odd67"], dict(ln=True, p=0.1), (0, 1)),     # 29 / 45 / 53 wide, a partial ln_bwd chunk
    "ln-wide1024": (LAYER_CASES["wide1024"], dict(ln=True), (0, 1)),        # 1024 / 400: ln_bwd's column loop, split-K
    "droq-split517": (LAYER_CASES["split517"], dict(ln=True, p=0.1), (0, 1)),   # 96 / 260, batch 517
    "ln-b2048": (LAYER_CASES["b2048"], dict(ln=True), (0, 1)),              # 128 ln_bwd chunks, 64 tasks, act_dim 8
    "droq-b2048": (LAYER_CASES["b2048"], dict(ln=True, p=0.05), (1,)),
    "ln-ms1280": (sp.ms_spec().to_json(), dict(ln=True), (1,)),             # the MTSAC learner: 3 x 400, batch 1280
    "ens3-odd67": (LAYER_CASES["odd67"], dict(E=3, ens=(1, "min")), (0, 1)),    # head_bwd_kernel in critic mode
    "ens10-b1": (LAYER_CASES["b1"], dict(E=10, ens=(10, "mean")), (0, 1)),
    "ens5-pdout257": (LAYER_CASES["pdout257"], dict(E=5, ens=(2, "min")), (0, 1)),     # policy_dout_kernel
    "ens3-pdout256": (LAYER_CASES["pdout256"], dict(E=3, ens=(3, "mean")), (0, 1)),    # the E-sum inside head_bwd
    "ens10-split517": (LAYER_CASES["split517"], dict(E=10, ens=(2, "min")), (0, 1)),   # > 24 problems per group
    "ens10-b2048": (LAYER_CASES["b2048"], dict(E=10, ens=(2, "mean")), (0, 1)),
    "ens5-vs1024-ln": (VS1024, dict(ln=True, E=5, ens=(2, "min")), (1,)),   # the VSAC learner's width and batch
    "rlpd": (RLPD, dict(ln=True, p=0.01, E=10, ens=(2, "min")), (0, 1)),    # RLPD / DroQ: E = 10, LayerNorm, dropout
    # precision 0 only: at precision 1 one of the fifteen head-bias gradients (a sum of 520 per-row TD errors) cancels to
    # 1/2471 of the sum of its terms' magnitudes on step 3, so the 3xTF32 rounding of Q (1.3e-6 per row, within REL) shows
    # there as 1.5e-4 (H100, measured); LayerNorm + DroQ + ensembles run at precision 1 in the one-replica rows
    "replicas": (REPLICA_SPEC, dict(ln=True, p=(0.05, 0.1, 0.2), E=5, ens=((1, "min"), (3, "mean"), (5, "min")), R=3),
                 (0,)),
}


def _spec(name):
    return sp.SacSpec(**CASES[name][0])


def _variant(name):
    v = dict(ln=False, p=None, E=2, ens=None, R=1)
    v.update(CASES[name][1])
    R = v["R"]
    per = lambda x: list(x) if isinstance(x, (list, tuple)) and len(x) == R and R > 1 else [x] * R    # noqa: E731
    v["rates"] = per(v["p"])
    v["ens_rows"] = [tuple(e) for e in per(v["ens"])] if v["ens"] is not None else [None] * R
    return v


# ---------------------------------------------------------------------------------------------------------------------
# the edges each case reaches, from its spec alone
# ---------------------------------------------------------------------------------------------------------------------
def edges(name):
    spec, v = _spec(name), _variant(name)
    B, A, hid = spec.batch, spec.act_dim, list(spec.critic_hidden)
    kinds = (["LN"] if v["ln"] and v["p"] is None else []) + (["DroQ"] if v["p"] is not None else []) + (
        ["E"] if v["E"] > 2 else [])
    have = set()
    for k in kinds:
        if B == 1:
            have.add(f"L1 {k}: batch 1")
        if B % LN_ROWS:
            have.add(f"L1 {k}: batch % 16")
        if B >= SPLIT_K_MIN:
            have.add(f"L4 {k}: batch >= 512")
        if B == 2048:
            have.add(f"L4 {k}: batch 2048")
        if spec.num_tasks == 64 and spec.weighted_loss:
            have.add(f"L6 {k}: 64 tasks, weighted")
        if A == 8:
            have.add(f"L6 {k}: act_dim 8")
        if k in ("LN", "DroQ"):
            if any(h > LN_THREADS for h in hid):
                have.add(f"L2 {k}: H > 256")
            if k == "DroQ" and any(h > 128 for h in hid):
                have.add("L2 DroQ: H > 128")
            if any(h % 4 and h % 32 for h in hid):
                have.add(f"L3 {k}: H % 4")
            if len(hid) == 1:
                have.add(f"L5 {k}: 1 hidden layer")
            if len(hid) >= 3:
                have.add(f"L5 {k}: 3 hidden layers")
    if v["E"] > 2:
        E = v["E"]
        if hid[-1] % 4 and E in (3, 10):
            have.add(f"E1: critic-mode head_bwd_kernel, E = {E}")
        have.add("E2: policy_dout_kernel" if B * A > 2048 else "E2: E-sum in head_bwd")
        if E == 10 and B >= SPLIT_K_MIN and set(CASES[name][2]) == {0, 1}:
            have.add("E3: E = 10 at batch >= 512, both precisions")
        for m, actor in v["ens_rows"]:
            have.add(f"E4: m = {'E' if m == E else m}")
            have.add(f"E4: {actor}")
        have.add(f"E4: E = {E}")
        if v["R"] == 3 and v["ln"] and v["p"] is not None and len(set(v["rates"])) == 3 and len(set(v["ens_rows"])) == 3:
            have.add("R: 3 replicas, LN + DroQ + E, own rates and (m, reduction)")
        if E == 10 and v["ln"] and v["p"] is not None and B == 256 and hid == [256] * len(hid):
            have.add("X: RLPD / DroQ at width 256, batch 256")
    return have


WANT = ({f"L1 {k}: {e}" for k in ("LN", "DroQ", "E") for e in ("batch 1", "batch % 16")}
        | {f"L2 {k}: H > 256" for k in ("LN", "DroQ")} | {"L2 DroQ: H > 128"}
        | {f"L3 {k}: H % 4" for k in ("LN", "DroQ")}
        | {f"L4 {k}: {e}" for k in ("LN", "DroQ", "E") for e in ("batch >= 512", "batch 2048")}
        | {f"L5 {k}: {e}" for k in ("LN", "DroQ") for e in ("1 hidden layer", "3 hidden layers")}
        | {f"L6 {k}: {e}" for k in ("LN", "E") for e in ("64 tasks, weighted", "act_dim 8")}
        | {"E1: critic-mode head_bwd_kernel, E = 3", "E1: critic-mode head_bwd_kernel, E = 10",
           "E2: policy_dout_kernel", "E2: E-sum in head_bwd", "E3: E = 10 at batch >= 512, both precisions",
           "E4: m = 1", "E4: m = 2", "E4: m = E", "E4: mean", "E4: min", "E4: E = 3", "E4: E = 5", "E4: E = 10",
           "R: 3 replicas, LN + DroQ + E, own rates and (m, reduction)", "X: RLPD / DroQ at width 256, batch 256"})


# ---- 5: the table reaches every edge (CPU) -----------------------------------------------------------------------------
def test_cases_reach_every_edge():
    have = set()
    for name in CASES:
        have |= edges(name)
    missing = sorted(WANT - have)
    assert not missing, f"no case reaches: {missing}"


def test_drop_masks_twin_tag_unchanged_and_ensemble_tags_distinct():
    """nets = 2 is the twin formula; an ensemble's E critics draw E distinct masks per (pass, layer)."""
    B, H, p = 5, 70, 0.3
    for pass_ in range(3):
        for l in range(3):
            for net in range(2):
                a = pr.drop_masks(9, 1, 4, pass_, l, net, B, H, p)
                b = pr.drop_masks(9, 1, 4, pass_, l, net, B, H, p, nets=2)
                assert np.array_equal(a, b)
    E = 10
    seen = {}
    for pass_ in range(3):
        for l in range(2):
            for k in range(E):
                m = pr.drop_masks(9, 1, 4, pass_, l, k, B, H, p, nets=E).tobytes()
                assert m not in seen, ((pass_, l, k), seen.get(m))
                seen[m] = (pass_, l, k)
    spec = sp.SacSpec(critic_hidden=[40, 33], batch=6)
    assert dq.step_masks(spec, 3, 2, p).keys() == dq.step_masks(spec, 3, 2, p, nets=2).keys()
    assert len(dq.step_masks(spec, 3, 2, p, nets=E)) == E * 3 * 2


def test_oracle_forced_min_equals_amin_when_nothing_is_forced():
    """amin_tagged without a forced mask (or with the mask of torch.amin's own choice) is torch.amin, value and gradient;
    forced onto a tie it splits the gradient evenly, as the library does."""
    g = torch.Generator().manual_seed(0)
    q = torch.randn(5, 7, 1, generator=g)
    q[2, 3] = q[4, 3] = q[:, 3].min() - 1.0                # an exact tie in row 3
    for forced in (None, "own"):
        a, b = q.clone().requires_grad_(), q.clone().requires_grad_()
        with sp.ReluTape() as tape:
            if forced == "own":
                tape.forced["amin:pi"] = (q - q.amin(0, keepdim=True)).reshape(5, 7) == 0
            ra = rq.amin_tagged(a, "amin:pi")
        rb = b.amin(0)
        assert torch.equal(ra, rb)
        ra.sum().backward()
        rb.sum().backward()
        assert torch.equal(a.grad, b.grad)
        assert a.grad[2, 3].item() == a.grad[4, 3].item() == 0.5
        assert (tape.z["amin:pi"] >= 0).all() and (tape.z["amin:pi"] == 0).sum() == 8
    # a forced critic the oracle would not take: its share of the gradient, and check_forced names it unless it is a tie
    m = (q - q.amin(0, keepdim=True)).reshape(5, 7) == 0
    m[0, 0] = True
    with sp.ReluTape({"amin:pi": m}) as tape:
        x = q.clone().requires_grad_()
        rq.amin_tagged(x, "amin:pi").sum().backward()
    assert x.grad[0, 0].item() > 0
    if tape.z["amin:pi"][0, 0] > 1e-3:
        with pytest.raises(AssertionError, match="amin:pi"):
            check_forced(tape, {"amin:pi": m})


# ---------------------------------------------------------------------------------------------------------------------
# handles, oracles and their state
# ---------------------------------------------------------------------------------------------------------------------
def _params(spec, E, ln, seed):
    """Xavier weights, small random biases, LayerNorm weights near 1 and biases near 0 (ln), targets equal to their
    locals, a temperature per task."""
    p = rq.init_params(spec, E, seed=seed) if E > 2 else sp.init_params(spec, seed=seed)
    g = torch.Generator().manual_seed(seed + 1000)
    for k in list(p):
        if k.endswith(".bias") and "_target." not in k:
            p[k] = 0.05 * torch.randn(p[k].shape, generator=g)
    if ln:
        for q in rq.nets(E):
            for l, H in enumerate(spec.critic_hidden):
                p[f"{q}.{l}.ln.weight"] = 1.0 + 0.1 * torch.randn(H, generator=g)
                p[f"{q}.{l}.ln.bias"] = 0.05 * torch.randn(H, generator=g)
    for k in list(p):
        if k.split(".")[0] in rq.nets(E):
            p[k.replace(".", "_target.", 1)] = p[k].clone()
    p["log_alpha"] = -0.5 + 0.5 * torch.randn(spec.n_alpha, generator=g)
    return p


class _EnsPort(rq.RedqPortLearner):
    """The ensemble oracle with LayerNorm (ln) and the philox_ref masks of the step it takes (p: DroQ)."""

    def __init__(self, spec, params, E, ens, ln, p, replica):
        super().__init__(spec, params, E, ens[0], ens[1], seed=SEED, replica=replica)
        self.ln, self.rate = ln, p

    def update_SAC(self, *args, **kw):
        if self.rate is not None:
            masks = dq.step_masks(self.spec, self.seed, self.step + 1, self.rate, self.replica, nets=self.E)
            ctx = rq.ensemble_dropout(masks, self.rate)
        else:
            ctx = lnp._layer_norm_mlp() if self.ln else contextlib.nullcontext()
        with ctx:
            return super().update_SAC(*args, **kw)


def _port(spec, v, r, params):
    if v["E"] > 2:
        return _EnsPort(spec, params, v["E"], v["ens_rows"][r], v["ln"], v["rates"][r], r)
    if v["rates"][r] is not None:
        return dq.DroqPortLearner(spec, params, v["rates"][r], SEED, replica=r)
    return lnp.LnPortLearner(spec, params)


def _core(spec, v, precision, R=None):
    from distributed_sac_b200.core import SacCore
    R = v["R"] if R is None else R
    kw = dict(critic_layer_norm=v["ln"], critic_dropout=v["p"] is not None)
    if v["E"] > 2:
        kw["critic_ensemble"] = v["E"]
    core = SacCore(core_config(spec, replicas=R, precision=precision, **kw), 0, seed=SEED)
    for r in range(R):
        if v["p"] is not None:
            core.set_critic_dropout(v["rates"][r], replica=r)
        if v["E"] > 2:
            core.set_ensemble(*v["ens_rows"][r], replica=r)
    return core


def _step_inputs(spec, R, i, seed=0):
    """Step i's minibatch and noise per replica."""
    gen = torch.Generator().manual_seed(seed + 50 + i)
    batches = [sp.synthetic_batch(spec, seed=seed + 300 + 10 * i + r) for r in range(R)]
    eps = [(torch.randn(spec.batch, spec.act_dim, generator=gen), torch.randn(spec.batch, spec.act_dim, generator=gen))
           for _ in range(R)]
    return batches, eps


def _run(core, batches, eps):
    core.step(*[torch.stack([b[j] for b in batches]) for j in range(5)], torch.stack([e[0] for e in eps]),
              torch.stack([e[1] for e in eps]))


def _row_outputs(E):
    return ROW_OUTPUTS if E == 2 else ("y",) + tuple(f"q{k + 1}" for k in range(E)) + ROW_OUTPUTS[2:]


def _mask_bits(core, spec, E, r):
    """{(letter, layer): bool [E][B][H]} of the replica's last step."""
    return {(k, l): core.debug(f"m{k}.{l}", r).reshape(E, spec.batch, H) == 1
            for k in KINDS for l, H in enumerate(spec.critic_hidden)}


def _check_labels(name, labels, precision):
    spec, v = _spec(name), _variant(name)
    B, E = spec.batch, v["E"]
    assert not any(l.startswith("chain") for l in labels), labels
    for pass_ in ("critic", "target", "actor pass"):
        for l in range(len(spec.critic_hidden)):
            assert (f"ln_fwd{{{pass_} {l}}}" in labels) == v["ln"], (pass_, l, labels)
    heads = [l for l in labels if l.startswith("head_bwd(q")]
    assert len(heads) == 2, labels
    slices = 4 if B >= SPLIT_K_MIN else 1
    assert all(l.endswith(f"row slices {slices})") for l in heads), heads
    if spec.critic_hidden[-1] % 4:
        assert not any("128-bit" in l for l in heads), heads
    assert ("policy_dout" in labels) == (B * spec.act_dim > 2048), labels
    if precision == 1 and B >= 128:
        assert any("wgmma" in l for l in labels), labels
    cut = [l for a, l in zip(labels, labels[1:]) if l == a and l.startswith("gemm_wgrad(") and "ffma" in l]
    if precision == 0 and E * 4 > GS_MAXG and B >= SPLIT_K_MIN:
        assert cut, f"no weight-gradient group cut into several launches: {labels}"


# ---- 1: step parity ----------------------------------------------------------------------------------------------------
PARITY = [(n, q) for n in CASES for q in CASES[n][2]]


@gpu
@pytest.mark.parametrize("name,precision", PARITY, ids=[f"{n}-p{q}" for n, q in PARITY])
def test_step_matches_oracle(cuda, name, precision):
    spec, v = _spec(name), _variant(name)
    R, E = v["R"], v["E"]
    core = _core(spec, v, precision)
    start = [_params(spec, E, v["ln"], seed=7 + 13 * r) for r in range(R)]
    ports = [_port(spec, v, r, start[r]) for r in range(R)]
    flips, worst, dropped = 0, 0.0, [0.0] * R
    routed = [False] * R
    for i in range(5):
        batches, eps = _step_inputs(spec, R, i)
        for r in range(R):
            sync_core_to_port(core, ports[r], r)
        _run(core, batches, eps)
        for r in range(R):
            what = f"{name} p{precision} step {i} replica {r}: "
            forced = cuda_relu_masks(core, spec, r, E=E)
            ref = capture_grads(ports[r])
            with sp.ReluTape(forced) as tape:
                o = ports[r].update_SAC(*batches[r], *eps[r], want_intermediates=True)
            flips += sum(check_forced(tape, forced, what).values())
            check_grads(core, ref, what, r)
            check_active(core, spec, r, what, E=E)
            check_losses(core, o, r, what)
            check_port_state(core, ports[r], r)
            worst = max(worst, check_rows(core, spec, o, r, what, _row_outputs(E)))
            if v["p"] is not None:
                dropped[r] += float(sum((~m).sum() for m in _mask_bits(core, spec, E, r).values()))
            if E > 2 and v["ens_rows"][r][1] == "min":
                routed[r] = routed[r] or bool((core.debug("dq_pi", r).reshape(E, -1)[1:] != 0).any())
    for r in range(R):
        got = core.get_named(PARAMS, r)
        for k in got:
            if k.split(".")[0] in rq.nets(E) or k.startswith("actor."):
                assert not torch.equal(got[k].reshape(-1), start[r][k].reshape(-1)), f"{name}: {k} of replica {r} did not move"
        if v["p"] is not None and v["rates"][r] > 0:
            assert dropped[r] > 0, f"{name}: replica {r} dropped nothing"
        if E > 2 and v["ens_rows"][r][1] == "min":
            assert routed[r], f"{name}: replica {r}'s min never routed to a critic other than critic 1"
    _check_labels(name, plan_labels(core), precision)
    core.close()
    print(f"[critic variants] {name} precision {precision}: {flips} kink flips, worst row deviation {worst:.2e}")


# ---- 2: the normalization launches alone ---------------------------------------------------------------------------------
NORM = ["ln-b1", "droq-b1", "droq-odd67", "droq-split517", "ln-wide1024", "rlpd", "replicas"]


@gpu
@pytest.mark.parametrize("precision", [0, 1])
@pytest.mark.parametrize("name", NORM)
def test_normalization_matches_fp64(cuda, name, precision):
    spec, v = _spec(name), _variant(name)
    R, E, B = v["R"], v["E"], spec.batch
    core = _core(spec, v, precision)
    before = [_params(spec, E, True, seed=5 + r) for r in range(R)]
    for r in range(R):
        core.set_named(before[r], PARAMS, r)
    _run(core, *_step_inputs(spec, R, 0))
    for r in range(R):
        after = core.get_named(PARAMS, r)
        # hQ / hT were normalized with the parameters before the step's updates, hP with the updated critics
        for kind, src, suffix in (("Q", before[r], ""), ("T", before[r], "_target"), ("P", after, "")):
            for l, H in enumerate(spec.critic_hidden):
                z = core.debug(f"z{kind}.{l}", r).reshape(E, B, H).double().numpy()
                h = core.debug(f"h{kind}.{l}", r).reshape(E, B, H).double().numpy()
                for k in range(E):
                    net = f"q{k + 1}{suffix}"
                    ref, _, _ = lnp.ln_forward(z[k], src[f"{net}.{l}.ln.weight"].reshape(-1).double().numpy(),
                                               src[f"{net}.{l}.ln.bias"].reshape(-1).double().numpy())
                    err = np.abs(h[k] - ref) / np.maximum(np.abs(ref), 1.0)
                    assert err.max() <= 1e-6, (name, r, kind, l, k, float(err.max()))
    core.close()


# ---- 3: the masks bit for bit ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("E", [2, 3, 10])
def test_masks_equal_philox_reference(cuda, E):
    """critic hidden widths 45 (% 32 != 0) and 260 (> 128), three replicas at their own rates; steps 1 and 3 are
    critic-only (actor interval 2): step 1 draws no actor-pass masks (the buffer keeps its zeros), step 3 leaves step 2's."""
    spec = sp.SacSpec(state_dim=9, act_dim=3, actor_hidden=[64, 64], critic_hidden=[45, 260], batch=67)
    rates = (0.05, 0.1, 0.5)
    v = dict(ln=True, p=rates, E=E, R=3, rates=list(rates), ens_rows=[(2, "mean")] * 3)
    core = _core(spec, v, 0)
    core.set_update_intervals(2, 1)
    B, last = spec.batch, None
    for step in range(1, 4):
        _run(core, *_step_inputs(spec, 3, step))
        now = {r: _mask_bits(core, spec, E, r) for r in range(3)}
        for r in range(3):
            for (kind, l), got in now[r].items():
                H = spec.critic_hidden[l]
                for k in range(E):
                    if kind == "P" and step != 2:
                        want = np.zeros((B, H), bool) if step == 1 else last[r][(kind, l)][k].numpy()
                    else:
                        want = pr.drop_masks(SEED, r, step, KINDS[kind], l, k, B, H, rates[r], nets=E)
                    assert np.array_equal(got[k].numpy(), want), (E, step, r, kind, l, k, int((got[k].numpy() != want).sum()))
        last = now
    core.close()


# ---- 4: replica independence ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["ln-b2048", "ens10-ln-split517"])
def test_replica_equals_single_handle(cuda, name):
    """Replica r of an R = 3 handle equals an R = 1 handle given replica r's state and inputs, bit for bit, at precision 0
    (the target subset is the full set, which does not depend on the replica's key)."""
    from distributed_sac_b200 import _lib
    if name == "ln-b2048":
        spec, v = _spec("ln-b2048"), _variant("ln-b2048")
    else:
        spec = sp.SacSpec(**LAYER_CASES["split517"])
        v = dict(ln=True, p=None, E=10, R=3, rates=[None] * 3, ens_rows=[(10, "min")] * 3)
    R, E = 3, v["E"]
    params = [_params(spec, E, True, seed=40 + r) for r in range(R)]
    many = _core(spec, v, 0, R=R)
    for r in range(R):
        many.set_named(params[r], PARAMS, r)
    steps = [_step_inputs(spec, R, i, seed=7) for i in range(2)]
    for batches, eps in steps:
        _run(many, batches, eps)
    for r in range(R):
        single = _core(spec, dict(v, rates=v["rates"][r:r + 1], ens_rows=v["ens_rows"][r:r + 1]), 0, R=1)
        single.set_named(params[r], PARAMS)
        for batches, eps in steps:
            _run(single, batches[r:r + 1], eps[r:r + 1])
        for which in (PARAMS, ADAM_M, ADAM_V, GRADS):
            a, b = many.get_named(which, r), single.get_named(which)
            diff = [k for k in a if not torch.equal(a[k], b[k])]
            assert not diff, f"{name}: replica {r} differs from the R = 1 handle in arena {which}: {diff[:8]}"
        assert torch.equal(many.read_losses(2)[:, r], single.read_losses(2)[:, 0]), r
        if r == R - 1:
            assert plan_labels(many) == plan_labels(single), "the R = 3 and R = 1 handles run different plans"
        single.close()
    many.close()
