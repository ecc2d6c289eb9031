"""Every Adam step, bit for bit, and the gradients it reads against the autograd oracle.

One Adam step moves an element by at most about lr (3e-4 here), about 0.5 % of a Xavier weight's norm: the 1e-4
relative-L2 bar of the parity tests accepts an error of up to ~2 % of the update, and a larger one on a few elements.  No
bar is needed.  The library is built with -fmad=false and without fast-math, and every writer of the update -- adam_kernel
of the per-layer and CARE plans (split-K gradient slices added in index order, replica strides, counter slots 0 critic,
1 actor, 4 CARE(O) context encoder), the fused optimizer epilogue of the layer-chained plan's wgrad_kernel (float4 body,
bias rows), the temperature Adam of the TAIL_ALPHA_AND_LOSSES job -- evaluates adam_scalars / adam_one with one rounding
per operation, in source order, from readable state: p, m, v before the step, the gradient it consumed (GRADS after the
step; b200sac_export adds the split-K slices in adam_kernel's order), the replica's learning rate and the fp64 bias
corrections Counters::b1p / b2p.  The counters are modelled here as the library keeps them: pow(beta, t) after
b200sac_set_steps, then one multiplication by beta per step that advances the slot (critic-only steps skip the actor and
the temperature).  So every trainable element must equal adam_expect() of its own slot as a bit pattern, and the gaps
between tensors must not change.  A failing tensor is tested against the mistakes that would explain it (another slot's
rate or count, another replica's row, t - 1 / t + 1, the gradient without its split-K slices, fp64 or FMA evaluation), and
the message names the one that reproduces it.

Bit-exactness on top of wrong gradients would prove nothing, so the first checked step of every plan also compares GRADS
with the gradients the oracle's optimizers consume (captured at each optimizer's step(), CUDA masks forced) at 1e-4 per
tensor.  The CPU test at the end ties adam_expect to torch.optim.Adam, the reference's optimizer.
"""
import math

import numpy as np
import pytest
import torch

import care_port as cp
import sac_port as sp
import test_gpu_targets_exact as te
from _golden import REL, care_core_config, core_config, kink_checked_step, rel_l2
from test_gpu_hparams import ROWS, _inputs
from test_gpu_targets_exact import LL_CFG, _bits, _learner, export

ADAM_M, ADAM_V, GRADS = 1, 2, 3
SLOT_OF_OPT = {0: 0, 1: 1, 2: 2, 3: 4}          # layout table "opt" -> Counters slot
LR_OF_SLOT = {0: "lr_critic", 1: "lr_actor", 2: "lr_alpha", 4: "lr_ctx"}
SLOT_NAME = {0: "critic", 1: "actor", 2: "temperature", 4: "context encoder"}

MT64 = dict(state_dim=17, num_tasks=64, act_dim=3, actor_hidden=[96, 80], critic_hidden=[72, 104], batch=320,
            weighted_loss=True)


# ---------------------------------------------------------------------------------------------------------------------
# the specification
# ---------------------------------------------------------------------------------------------------------------------
def adam_expect(p, m, v, g, lr, b1p, b2p, beta1=0.9, beta2=0.999, eps=1e-8, mode="fp32"):
    """(p', m', v') of adam_scalars + adam_one: step_size = f32(lr / (1 - b1p)) and bc2_sqrt = f32(sqrt(1 - b2p)) in fp64,
    then m' = m + w1*(g - m), v' = v*b2 + (omb2*g)*g, p' = p - step_size*(m' / (sqrtf(v')/bc2_sqrt + eps)), one fp32
    rounding per operation.  mode "fp64": the same formula evaluated in fp64 and rounded once; mode "fma": the multiply-adds
    contracted (the two diagnostics a failing element is tested against)."""
    f = np.float32
    step_size, bc2_sqrt = f(lr / (1.0 - b1p)), f(math.sqrt(1.0 - b2p))
    w1, b2, omb2, e = f(1.0 - beta1), f(beta2), f(1.0 - beta2), f(eps)
    p, m, v, g = (np.asarray(x, dtype=np.float32) for x in (p, m, v, g))
    if mode == "fp64":
        d = np.float64
        m1 = m + d(w1) * (g.astype(d) - m)
        v1 = v * d(b2) + (d(omb2) * g) * g
        p1 = p - d(step_size) * (m1 / (np.sqrt(v1) / d(bc2_sqrt) + d(e)))
        return p1.astype(f), m1.astype(f), v1.astype(f)
    if mode == "fma":
        d = np.float64
        m1 = (d(w1) * (g - m) + m).astype(f)
        v1 = ((omb2 * g).astype(d) * g + v * b2).astype(f)
        q = m1 / (np.sqrt(v1) / bc2_sqrt + e)
        return (p.astype(d) - d(step_size) * q).astype(f), m1, v1
    m1 = m + w1 * (g - m)
    v1 = v * b2 + (omb2 * g) * g
    p1 = p - step_size * (m1 / (np.sqrt(v1) / bc2_sqrt + e))
    return p1, m1, v1


class Counts:
    """fp64 model of one replica's Counters: Adam step and bias-correction products per slot (0 critic, 1 actor,
    2 temperature, 4 context encoder)."""

    def __init__(self, beta1, beta2):
        self.beta1, self.beta2 = beta1, beta2
        self.t, self.b1p, self.b2p = [0] * 5, [1.0] * 5, [1.0] * 5

    def seed(self, steps):
        """b200sac_set_steps: (critic, actor, alpha, context encoder) -> glibc pow, as on the host side"""
        for i, s in enumerate(steps):
            slot = 4 if i == 3 else i
            self.t[slot] = int(s)
            self.b1p[slot], self.b2p[slot] = math.pow(self.beta1, s), math.pow(self.beta2, s)

    def bump(self, actor_every=1):
        """bump_counters: every slot but actor and temperature on a critic-only step; returns 'actor step'."""
        n = self.t[0] + 1
        act = actor_every == 1 or n % actor_every == 0
        for i in range(5):
            if act or i not in (1, 2):
                self.t[i] += 1
                self.b1p[i] *= self.beta1
                self.b2p[i] *= self.beta2
        return act

    def copy(self):
        c = Counts(self.beta1, self.beta2)
        c.t, c.b1p, c.b2p = list(self.t), list(self.b1p), list(self.b2p)
        return c

    def steps(self, n):
        return tuple(self.t[i] for i in (0, 1, 2, 4))[:n]


def new_model(core):
    return [Counts(core.cfg.beta1, core.cfg.beta2) for _ in range(core.cfg.replicas)]


def set_steps(core, model, r, steps):
    core.set_steps(steps, r)
    got = core.get_steps(r)
    model[r].seed(list(got) + [0] * (4 - len(got)))      # set_steps reseeds every slot it does not name from its count


# ---------------------------------------------------------------------------------------------------------------------
# the check
# ---------------------------------------------------------------------------------------------------------------------
def _slots(core):
    """(slot of every trainable float, -1 in the gaps; [(name, offset, floats, slot)] of the trainable tensors)"""
    if not hasattr(core, "_adam_slots"):
        slot = np.full(core.trainable_floats, -1, np.int8)
        tensors = []
        for name, (off, rows, _cols, tr, opt, pitch) in core.table.items():
            if tr:
                slot[off:off + rows * pitch] = SLOT_OF_OPT[opt]
                tensors.append((name, off, rows * pitch, SLOT_OF_OPT[opt]))
        core._adam_slots = (slot, tensors)
    return core._adam_slots


def snapshot(core, r, with_grads=False):
    """(p[:trainable], m, v[, GRADS]) of replica r as numpy arrays"""
    T = core.trainable_floats
    out = [export(core, r)[:T], core.export_arena(ADAM_M, r).numpy().copy(), core.export_arena(ADAM_V, r).numpy().copy()]
    if with_grads:
        out.append(core.export_arena(GRADS, r).numpy().copy())
    return out


def _slice0(core, r):
    """The gradient arena without the extra split-K slices (b200sac_read_range reads slice 0 only)."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import _ptr, _stream
    out = torch.empty(core.trainable_floats)
    _lib.check(core.lib.b200sac_read_range(core._h, GRADS, r, 0, core.trainable_floats, _ptr(out), _stream()))
    return out.numpy()


def _candidates(core, model, r, s, before, g, sel):
    """{mistake: (p', m', v')} for the elements sel of slot s of replica r"""
    cfg, c = core.cfg, model[r]
    hp = core.get_hparams(r)
    pb, mb, vb = (x[sel] for x in before)
    ex = lambda lr, b1p, b2p, gg=None, mode="fp32": None if b1p >= 1.0 else adam_expect(    # (count 0: no step uses it)
        pb, mb, vb, g[sel] if gg is None else gg, lr, b1p, b2p, cfg.beta1, cfg.beta2, cfg.adam_eps, mode)
    lr, b1p, b2p = hp[LR_OF_SLOT[s]], c.b1p[s], c.b2p[s]
    out = {"no update": (pb, mb, vb)}
    for s2 in (0, 1, 2, 4):
        if s2 != s:
            out[f"the {SLOT_NAME[s2]} slot's rate and count"] = ex(hp[LR_OF_SLOT[s2]], c.b1p[s2], c.b2p[s2])
            out[f"the {SLOT_NAME[s2]} slot's count"] = ex(lr, c.b1p[s2], c.b2p[s2])
    for q in range(cfg.replicas):
        if q != r:
            out[f"replica {q}'s {LR_OF_SLOT[s]}"] = ex(core.get_hparams(q)[LR_OF_SLOT[s]], b1p, b2p)
            out[f"replica {q}'s count"] = ex(lr, model[q].b1p[s], model[q].b2p[s])
    out["count t - 1"] = ex(lr, b1p / cfg.beta1, b2p / cfg.beta2)
    out["count t + 1"] = ex(lr, b1p * cfg.beta1, b2p * cfg.beta2)
    out["pow(beta, t) instead of the running product"] = ex(lr, math.pow(cfg.beta1, c.t[s]), math.pow(cfg.beta2, c.t[s]))
    out["the gradient without its split-K slices"] = ex(lr, b1p, b2p, _slice0(core, r)[sel])
    out["fp64 evaluation"] = ex(lr, b1p, b2p, mode="fp64")
    out["FMA-contracted evaluation"] = ex(lr, b1p, b2p, mode="fma")
    return {k: c for k, c in out.items() if c is not None}


def check_adam(core, model, r, before, after, act, what):
    """Every trainable element of replica r after one step == adam_expect of its slot (actor and temperature untouched on
    a critic-only step), p, m and v bit for bit; the gaps between tensors unchanged.  model[r] holds the counters the step
    used (bumped).  Returns {slot: elements whose parameter moved}."""
    cfg = core.cfg
    slot, tensors = _slots(core)
    hp = core.get_hparams(r)
    got = after[:3]
    g = after[3]
    want = [np.empty_like(x) for x in before]
    for s in (0, 1, 2, 4):
        sel = slot == s
        if not sel.any():
            continue
        if s in (1, 2) and not act:
            res = [x[sel] for x in before]
        else:
            res = adam_expect(before[0][sel], before[1][sel], before[2][sel], g[sel], hp[LR_OF_SLOT[s]], model[r].b1p[s],
                              model[r].b2p[s], cfg.beta1, cfg.beta2, cfg.adam_eps)
        for w, x in zip(want, res):
            w[sel] = x
    gap = slot < 0
    for w, b in zip(want, before):
        w[gap] = b[gap]
    bad = []
    for name, off, n, s in tensors:
        sl = slice(off, off + n)
        diff = np.zeros(n, bool)
        for x, w in zip(got, want):
            diff |= _bits(x[sl]) != _bits(w[sl])
        if not diff.any():
            continue
        sel = np.zeros(core.trainable_floats, bool)
        sel[sl] = True
        cands = _candidates(core, model, r, s, before, g, sel)
        hit = [k for k, c in cands.items() if all(np.array_equal(_bits(x[sl]), _bits(y)) for x, y in zip(got, c))]
        i = int(np.argmax(diff))
        bad.append(f"{name} ({SLOT_NAME[s]} slot, t = {model[r].t[s]}, {LR_OF_SLOT[s]} = {hp[LR_OF_SLOT[s]]}; it got "
                   f"{' / '.join(hit) or 'no candidate'}): {int(diff.sum())} of {n} elements differ, first [{i}] "
                   f"g = {g[off + i]!r}: (p, m, v) = {tuple(float(x[off + i]) for x in got)} want "
                   f"{tuple(float(w[off + i]) for w in want)}")
    assert not bad, f"{what}: " + "; ".join(bad[:6])
    changed = gap & ((_bits(got[0]) != _bits(before[0])) | (_bits(got[1]) != _bits(before[1])) |
                     (_bits(got[2]) != _bits(before[2])))
    assert not changed.any(), f"{what}: {int(changed.sum())} floats between tensors changed, first [{int(np.argmax(changed))}]"
    return {s: int(((slot == s) & (got[0] != before[0])).sum()) for s in (0, 1, 2, 4) if (slot == s).any()}


def plant_edges(core, r):
    """Three real elements per trainable tensor: m = v = 0 (a fresh element), a denormal v, a tiny m."""
    m, v = core.export_arena(ADAM_M, r).numpy().copy(), core.export_arena(ADAM_V, r).numpy().copy()
    for name, (off, rows, cols, tr, _o, pitch) in core.table.items():
        if not tr:
            continue
        n = rows * cols
        for j, (mm, vv) in enumerate(((0.0, 0.0), (None, 1e-41), (1e-30, None))):
            r_, c_ = divmod((j * (n // 3 + 1) + 1) % n, cols)
            i = off + r_ * pitch + c_
            if mm is not None:
                m[i] = mm
            if vv is not None:
                v[i] = vv
    core.import_arena(torch.from_numpy(m), ADAM_M, r)
    core.import_arena(torch.from_numpy(v), ADAM_V, r)


def checked_steps(core, spec, care, model, n_steps, what, step_fn=None, actor_every=1, first=0):
    """n_steps steps (default: b200sac_step on _inputs), each replica checked after each; returns {slot: moved elements}
    summed over replicas and steps, and the actor steps seen per replica."""
    R = core.cfg.replicas
    moved, acts = {}, [0] * R
    for i in range(n_steps):
        before = [snapshot(core, r) for r in range(R)]
        if step_fn is None:
            b, e1, e2 = _inputs(spec, care, R, first + i)
            core.step(*b, e1, e2)
        else:
            step_fn(i)
        for r in range(R):
            act = model[r].bump(actor_every)
            acts[r] += act
            assert core.get_steps(r) == model[r].steps(len(core.get_steps(r))), (what, i, r)
            for s, k in check_adam(core, model, r, before[r], snapshot(core, r, True), act,
                                   f"{what} step {i} replica {r}").items():
                moved[s] = moved.get(s, 0) + k
    return moved, acts


def assert_moved(moved, care_o, what):
    want = (0, 1, 2) + ((4,) if care_o else ())
    assert all(moved.get(s, 0) > 0 for s in want), f"{what}: a slot never moved a parameter ({moved}): the case is vacuous"


# ---------------------------------------------------------------------------------------------------------------------
# the oracle's gradients
# ---------------------------------------------------------------------------------------------------------------------
def _port_of(core, spec, care, r=0):
    """An oracle learner holding replica r's state, rates and counts."""
    named = core.get_named(0, r)
    st = {"m": core.get_named(ADAM_M, r), "v": core.get_named(ADAM_V, r), "step": core.get_steps(r)}
    port = cp.CarePortLearner(spec, named, st) if care else sp.PortLearner(spec, named, st)
    hp = core.get_hparams(r)
    for opt, key in ((port.opt_critic, "lr_critic"), (port.opt_actor, "lr_actor"), (port.opt_alpha, "lr_alpha"),
                     (getattr(port, "opt_ctx", None), "lr_ctx")):
        if opt is not None:
            for grp in opt.param_groups:
                grp["lr"] = hp[key]
    return port


def capture_grads(port):
    """{name: gradient} as each optimizer's step() consumes it (the critic's before pi_loss.backward() adds to it)."""
    grads = {}
    names = {id(t): k for k, t in port.p.items()}
    for opt in (port.opt_critic, port.opt_actor, port.opt_alpha, getattr(port, "opt_ctx", None)):
        if opt is None:
            continue

        def step(*a, _opt=opt, _orig=opt.step, **kw):
            for grp in _opt.param_groups:
                for t in grp["params"]:
                    grads[names[id(t)]] = torch.zeros_like(t) if t.grad is None else t.grad.detach().clone()
            return _orig(*a, **kw)
        opt.step = step
    return grads


def check_grads(core, ref, what, r=0):
    """GRADS == the oracle's consumed gradients to 1e-4 per tensor (log_alpha: or 1e-6 absolute)."""
    got = core.get_named(GRADS, r)
    bad = []
    for k, g in got.items():
        assert k in ref, f"{what}: the oracle has no gradient for {k}"
        err = rel_l2(g, ref[k].reshape(g.shape))
        if err > REL and not (k == "log_alpha" and float((g - ref[k].reshape(g.shape)).abs().max()) <= 1e-6):
            bad.append((k, float(f"{err:.2e}")))
    assert not bad, f"{what}: gradients differ from the oracle's beyond {REL} (CUDA masks forced): {bad[:8]}"
    return len(got)


def oracle_checked_step(core, spec, care, model, i, what):
    """One step of replica 0 checked twice: GRADS against the oracle's consumed gradients, and the update exactly."""
    port = _port_of(core, spec, care)
    ref = capture_grads(port)
    set_steps(core, model, 0, core.get_steps(0))     # kink_checked_step reseeds the counters from the oracle's counts
    before = snapshot(core, 0)
    b, e1, e2 = _inputs(spec, care, 1, 100 + i)
    kink_checked_step(core, port, spec, [x[0] for x in b], e1[0], e2[0], care=care)
    act = model[0].bump()
    after = snapshot(core, 0, True)
    check_grads(core, ref, what)
    return check_adam(core, model, 0, before, after, act, what)


# ---------------------------------------------------------------------------------------------------------------------
# 1: every plan and writer: counts of their own per slot, edge elements, gradients against the oracle
# ---------------------------------------------------------------------------------------------------------------------
SAC_PLANS = ["chained_ll", "chained_deep8", "chained_big_odd", "vs400_fp32", "vs400_tc", "split517_fp32", "split517_tc",
             "wide1024_tc", "mtsac_t10", "mtsac_t64"]
PLANS = SAC_PLANS + ["care_m", "care_o"]


@pytest.fixture(scope="module")
def cuda():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from distributed_sac_b200 import _lib
    _lib.load()
    return torch.device("cuda", 0)


def _make(name, R=1, rows=None):
    """(core, spec, care): test_gpu_targets_exact's plans and parameters (targets off their locals), plus MTSAC at T = 64;
    each replica its own parameters and, if given, its own hyperparameter row."""
    from distributed_sac_b200.core import SacCore
    spec, care, precision = (sp.SacSpec(**MT64), False, 1) if name == "mtsac_t64" else te._plan(name)
    core = SacCore((care_core_config if care else core_config)(spec, replicas=R, precision=precision), 0, seed=0)
    for r in range(R):
        core.set_named(te._params(spec, care, seed=11 + 7 * r), 0, r)
        if rows is not None:
            core.set_hparams(r, **rows[r])
    return core, spec, care


@pytest.mark.gpu
@pytest.mark.parametrize("name", PLANS)
def test_adam_is_exact(cuda, name):
    core, spec, care = _make(name)
    care_o = care and core.cfg.care_original
    model = new_model(core)
    checked_steps(core, spec, care, model, 2, f"{name} warm-up")
    set_steps(core, model, 0, (7, 1, 10 ** 6, 3))
    plant_edges(core, 0)
    moved = oracle_checked_step(core, spec, care, model, 0, f"{name} oracle step")
    more, _ = checked_steps(core, spec, care, model, 2, name, first=10)
    for s, k in more.items():
        moved[s] = moved.get(s, 0) + k
    assert_moved(moved, care_o, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: three replicas, each its own rates (one at lr = 0) and its own counts 0, 1, 7, 10^6 per slot
# ---------------------------------------------------------------------------------------------------------------------
R3_PLANS = ["chained_ll", "chained_big_odd", "vs400_tc", "split517_fp32", "mtsac_t10", "care_m", "care_o"]
R3_COUNTS = [(10 ** 6, 7, 1, 0), (1, 0, 7, 10 ** 6), (7, 10 ** 6, 0, 1)]   # replica 1 trains at lr = 0


@pytest.mark.gpu
@pytest.mark.parametrize("name", R3_PLANS)
def test_adam_is_exact_per_replica(cuda, name):
    rows = [dict(ROWS[0]), dict(ROWS[1], lr_critic=0.0, lr_actor=0.0, lr_alpha=0.0, lr_ctx=0.0), dict(ROWS[2])]
    core, spec, care = _make(name, R=3, rows=rows)
    model = new_model(core)
    for r in range(3):
        set_steps(core, model, r, R3_COUNTS[r])
        plant_edges(core, r)
    p1 = snapshot(core, 1)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} R = 3")
    assert_moved(moved, care and core.cfg.care_original, name)
    after = snapshot(core, 1)
    assert np.array_equal(_bits(after[0]), _bits(p1[0])), "replica 1 (lr = 0) moved a parameter"
    assert not np.array_equal(after[1], p1[1]), "replica 1 (lr = 0) did not update its moments"
    assert model[0].b2p[0] == 0.0 and model[2].b2p[1] == 0.0, "b2p did not underflow at 10^6 steps"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: actor every 3rd, targets every 2nd step: the critic exact on every step, actor and temperature on actor steps
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "vs400_tc", "split517_fp32", "mtsac_t10", "care_o"])
def test_adam_is_exact_under_update_intervals(cuda, name):
    core, spec, care = _make(name, R=2, rows=ROWS[:2])
    core.set_update_intervals(actor_every=3, target_every=2)
    model = new_model(core)
    set_steps(core, model, 1, (4, 1, 1, 4))
    moved, acts = checked_steps(core, spec, care, model, 6, f"{name} actor_every = 3", actor_every=3)
    assert acts == [2, 2], f"expected two actor steps per replica in six, saw {acts}"
    assert_moved(moved, care and core.cfg.care_original, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: state carried over: copy_replica, a Learner checkpoint restore
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "split517_tc", "care_o"])
def test_adam_is_exact_after_copy_replica(cuda, name):
    core, spec, care = _make(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    checked_steps(core, spec, care, model, 2, f"{name} warm-up")
    set_steps(core, model, 0, (7, 1, 10 ** 6, 3))
    core.copy_replica(0, 1)
    model[1] = model[0].copy()
    assert core.get_steps(1) == core.get_steps(0)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} after copy_replica", first=20)
    assert_moved(moved, care and core.cfg.care_original, name)
    core.close()


@pytest.mark.gpu
def test_adam_is_exact_after_checkpoint_restore(cuda, tmp_path, monkeypatch):
    monkeypatch.chdir(tmp_path)
    a = _learner("LL", tmp_path)
    spec = sp.ll_spec(batch=LL_CFG["batch_size"])
    try:
        for i in range(3):
            b, e1, e2 = _inputs(spec, False, 1, i)
            a.core.step(*b, e1, e2)
        path = a.save_checkpoint(5)
    finally:
        a.memory.stop()
    lrn = _learner("LL", tmp_path)
    try:
        lrn.load_checkpoint(path)
        core = lrn.core
        assert core.get_steps() == (3, 3, 3)
        model = new_model(core)
        model[0].seed(list(core.get_steps()) + [0])         # load_checkpoint -> set_steps: pow(beta, t)
        moved, _ = checked_steps(core, spec, False, model, 2, "LL after load_checkpoint", first=30)
        assert_moved(moved, False, "checkpoint restore")
    finally:
        lrn.memory.stop()


# ---------------------------------------------------------------------------------------------------------------------
# 5: the other entry points: step_sampled from a device ring (graph path), step_host
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("name", ["chained_ll", "split517_tc", "care_o"])
def test_sampled_step_adam_is_exact(cuda, name):
    from distributed_sac_b200.core import Replay
    core, spec, care = _make(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    set_steps(core, model, 1, (7, 1, 10 ** 6, 3))
    cap = 4 * spec.batch * max(spec.num_tasks, 1)
    ring = Replay(core, cap, "device", seed=5)
    ring.fill_synthetic(cap, seed=6)
    moved, _ = checked_steps(core, spec, care, model, 3, f"{name} step_sampled", step_fn=lambda i: core.step_sampled(ring, 1))
    assert_moved(moved, care and core.cfg.care_original, name)
    ring.close()
    core.close()


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["vs400_fp32"])
def test_host_step_adam_is_exact(cuda, name):
    core, spec, care = _make(name, R=2, rows=ROWS[:2])
    model = new_model(core)
    set_steps(core, model, 0, (7, 1, 10 ** 6))

    def step(i):
        b, e1, e2 = _inputs(spec, care, 2, 40 + i)
        core.step_host(*b, e1, e2)
    moved, _ = checked_steps(core, spec, care, model, 2, f"{name} step_host", step_fn=step)
    assert_moved(moved, False, name)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 6 (CPU): the specification against the reference's optimizer
# ---------------------------------------------------------------------------------------------------------------------
def test_adam_expect_follows_torch_adam():
    """adam_expect against torch.optim.Adam (CPU defaults) over six steps of random fp32 state with tiny and zero
    gradients.  torch contracts lerp_ / addcmul_ into FMAs, so m and v may differ in the last bits; p must agree to
    1e-3 of the update bound lr, m and v to a few ulp of the magnitudes they are formed from."""
    lr, beta1, beta2, eps = 3e-4, 0.9, 0.999, 1e-8
    rng = np.random.default_rng(7)
    n = 200_000
    p0 = (rng.standard_normal(n) * 0.0625).astype(np.float32)
    param = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([param], lr=lr, betas=(beta1, beta2), eps=eps)
    p, m, v = p0.copy(), np.zeros(n, np.float32), np.zeros(n, np.float32)
    ulp = np.finfo(np.float32).eps
    differ = 0
    for t in range(1, 7):
        g = (rng.standard_normal(n) * 10.0 ** rng.uniform(-8, 0, n)).astype(np.float32)
        g[rng.random(n) < 0.05] = 0.0
        g[rng.random(n) < 0.02] = np.float32(1e-30) * rng.standard_normal()
        param.grad = torch.from_numpy(g.copy())
        opt.step()
        scale_m = np.abs(m) + np.abs(g) * np.float32(1 - beta1)
        scale_v = np.abs(v) + np.float32(1 - beta2) * g * g
        p, m, v = adam_expect(p, m, v, g, lr, beta1 ** t, beta2 ** t, beta1, beta2, eps)
        st = opt.state[param]
        tm, tv, tp = st["exp_avg"].numpy(), st["exp_avg_sq"].numpy(), param.detach().numpy()
        assert np.abs(tp.astype(np.float64) - p).max() <= 1e-3 * lr, t
        assert (np.abs(tm.astype(np.float64) - m) <= 2 * ulp * scale_m).all(), t
        assert (np.abs(tv.astype(np.float64) - v) <= 2 * ulp * scale_v).all(), t
        differ += int((tm != m).sum())
        # keep the two trajectories from drifting apart: continue from torch's state
        p, m, v = tp.copy(), tm.copy(), tv.copy()
    assert differ > 0, "torch and adam_expect agree bit for bit: the bars are not exercised"
