"""GPU: every write of the target networks, bit for bit.

A Polyak step moves a target by tau * (local - target), about 1e-5 of its norm at tau = 0.005: a relative-L2 bar of 1e-4
cannot see a target blended from the pre-Adam local, with another replica's rate, or with tau instead of tau_se.  None
is needed either.  The library is built with -fmad=false, and every writer of a target -- the fused optimizer tile of
the layer-chained plan (chain.cuh, float4 body and bias rows), adam_kernel of the per-layer and CARE plans (split-K
slices, the switch from tau to tau_se at the CARE state encoder, the target schedule), polyak_kernel behind
b200sac_soft_update / b200sac_soft_update_critic -- computes fl(fl(ta * p) + fl(tb * t)) with (ta, tb) = ((float)tau,
(float)(1 - tau)), p the local it has just stored and t the target before the step.  That is the reference's
tau*local + (1.0-tau)*target on fp32 tensors (LL/learner.py:126-137), and it is fully determined by readable state: the
locals after the step and the targets before it.  So every element of q1_target.*, q2_target.* and tse.* (pad columns of
padded first layers included) must equal that expectation as a bit pattern, and nothing else outside the trainable prefix
(the CARE embedding, the gaps between tensors) may change at all.
"""
import numpy as np
import pytest
import torch

from _harness import PARAMS, ROWS, _bits, _handle, _inputs, _learner, cuda, export

pytestmark = pytest.mark.gpu

# _harness.SAC_PLANS / CARE_PLANS ids.  Chained: the LL shape, width-4 layers with 8 hidden layers, batch 531.
# Per-layer: fp32 FFMA and wgmma 3xTF32 at 400 wide; split-K weight-gradient slices and K tails (split517, wide1024).
PLANS = ["chained_ll", "chained_deep8", "chained_big_odd", "vs400_fp32", "vs400_tc", "split517_fp32", "split517_tc",
         "wide1024_tc", "mtsac_t10", "care_m", "care_o"]
# the R = 3 cases: one per step plan
R3_PLANS = ["chained_ll", "chained_big_odd", "vs400_fp32", "vs400_tc", "split517_tc", "mtsac_t10", "care_m", "care_o"]


def target_pairs(core):
    """[(target tensor, local tensor, hyperparameter of its rate)]"""
    out = []
    for name in core.table:
        if name.startswith(("q1_target.", "q2_target.")):
            out.append((name, name.replace("_target.", ".", 1), "tau"))
        elif name.startswith("tse."):
            out.append((name, "cse." + name[4:], "tau_se"))
    return out


def polyak(local, target, tau):
    """fl(fl(ta * local) + fl(tb * target)) in fp32, (ta, tb) = ((float)tau, (float)(1 - tau)) -- one rounding per op."""
    return np.float32(tau) * local + np.float32(1.0 - tau) * target


def check_targets(core, before, after, rates, moved, what, others=()):
    """Every target element == polyak(local after, target before, its rate) bit for bit (moved), or == the target before
    (not moved); everything else outside the trainable prefix unchanged.  rates: {"tau": .., "tau_se": ..}; others: more
    rates a failing tensor is tested against, so that the message names the rate it actually got."""
    T = core.trainable_floats
    covered = np.zeros(core.arena_floats - T, dtype=bool)
    bad = []
    n_el = 0
    for tname, lname, key in target_pairs(core):
        off, rows, _cols, _tr, _opt, pitch = core.table[tname]
        loff = core.table[lname][0]
        n = rows * pitch
        t_old, got, l_new = before[off:off + n], after[off:off + n], after[loff:loff + n]
        want = polyak(l_new, t_old, rates[key]) if moved else t_old
        diff = _bits(got) != _bits(want)
        covered[off - T:off - T + n] = True
        n_el += n
        if diff.any():
            cands = {f"{k} = {v}": polyak(l_new, t_old, v) for k, v in list(rates.items()) + list(others)}
            cands["the target before the step (not written)"] = t_old
            got_rate = [k for k, c in cands.items() if np.array_equal(_bits(got), _bits(c))]
            if np.array_equal(_bits(got), _bits(polyak(before[loff:loff + n], t_old, rates[key]))):
                got_rate.append(f"{key} applied to the pre-step local")
            i = int(np.argmax(diff))
            bad.append(f"{tname} (expected {'rate ' + key + ' = ' + str(rates[key]) if moved else 'untouched'}; it got "
                       f"{' / '.join(got_rate) or 'no candidate rate'}): {int(diff.sum())} of {n} elements differ, first "
                       f"[{i}] got {got[i]!r} want {want[i]!r}")
    assert not bad, f"{what}: " + "; ".join(bad[:6])
    rest = ~covered
    changed = rest & (_bits(after[T:]) != _bits(before[T:]))
    if changed.any():
        i = int(np.argmax(changed)) + T
        owner = [k for k, d in core.table.items() if d[0] <= i < d[0] + d[1] * d[5]]
        raise AssertionError(f"{what}: {int(changed.sum())} floats outside the targets changed, first arena[{i}] ({owner})")
    return n_el


def _plant_negative_zeros(core, replica=0, per_tensor=4):
    """A few -0.0 target elements per tensor (real columns): a writer that touches a target it must not, or uses another
    formula than the reference's, changes their sign."""
    a = core.export_arena(PARAMS, replica)
    for tname, _l, _k in target_pairs(core):
        off, rows, cols, _tr, _opt, pitch = core.table[tname]
        for j in range(min(per_tensor, rows * cols)):
            r_, c_ = divmod((j * 7919) % (rows * cols), cols)
            a[off + r_ * pitch + c_] = -0.0
    core.import_arena(a, PARAMS, replica)


def _rates(core, r):
    hp = core.get_hparams(r)
    return {"tau": hp["tau"], "tau_se": hp["tau_se"]}


def _other_rates(core, r):
    return [(f"replica {q}'s {k}", v) for q in range(core.cfg.replicas) if q != r for k, v in _rates(core, q).items()]


def run_checked_steps(core, spec, care, n_steps, what, target_every=1):
    R = core.cfg.replicas
    targets_moved = 0
    for i in range(n_steps):
        before = [export(core, r) for r in range(R)]
        b, e1, e2 = _inputs(spec, care, R, i)
        core.step(*b, e1, e2)
        for r in range(R):
            n = core.get_steps(r)[0]
            moved = n % target_every == 0
            targets_moved += moved
            check_targets(core, before[r], export(core, r), _rates(core, r), moved, f"{what} step {i} replica {r}",
                          _other_rates(core, r))
    return targets_moved


# ---------------------------------------------------------------------------------------------------------------------
# 1: the step's own target writes, every plan, one replica and three with hyperparameter rows of their own
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", PLANS)
def test_step_targets_are_exact(cuda, name):
    core, spec, care = _handle(name)
    if care:
        hp = core.get_hparams(0)
        assert hp["tau"] != hp["tau_se"], hp
    _plant_negative_zeros(core)
    run_checked_steps(core, spec, care, 3, name)
    core.close()


@pytest.mark.parametrize("name", R3_PLANS)
def test_step_targets_are_exact_per_replica(cuda, name):
    """Three replicas, each its own parameters, minibatches and hyperparameter row (every tau and tau_se differs): each
    replica's targets follow its own rates."""
    core, spec, care = _handle(name, R=3, rows=ROWS)
    assert len({r["tau"] for r in ROWS}) == 3 and len({r["tau_se"] for r in ROWS}) == 3
    run_checked_steps(core, spec, care, 2, f"{name} R = 3")
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 2: target update interval -- the formula on target steps, not a bit changed on the others
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", ["chained_ll", "vs400_tc", "split517_fp32", "care_m"])
def test_target_interval_writes_only_on_target_steps(cuda, name):
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    core.set_update_intervals(target_every=3)
    for r in range(2):
        _plant_negative_zeros(core, r)
    moved = run_checked_steps(core, spec, care, 7, f"{name} target_every = 3", target_every=3)
    assert moved == 2 * 2, f"expected target steps 3 and 6 on both replicas, saw {moved} target updates"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 3: sampled steps (in-kernel noise, device sampler), one step per call; a prioritized ring
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,prioritized", [("chained_ll", False), ("vs400_tc", False), ("care_o", False),
                                              ("split517_fp32", True)], ids=["chained_ll", "vs400_tc", "care_o", "per_split517"])
def test_sampled_step_targets_are_exact(cuda, name, prioritized):
    from distributed_sac_b200.core import Replay
    core, spec, care = _handle(name, R=2, rows=ROWS[:2])
    per = dict(alpha=0.6, beta=0.4, eps=1e-6) if prioritized else None
    cap = 4 * spec.batch * max(spec.num_tasks, 1)
    ring = Replay(core, cap, "device", seed=5, prioritized=per)
    ring.fill_synthetic(cap, seed=6)
    for i in range(3):
        before = [export(core, r) for r in range(2)]
        core.step_sampled(ring, 1)
        for r in range(2):
            check_targets(core, before[r], export(core, r), _rates(core, r), True, f"{name} sampled step {i} replica {r}",
                          _other_rates(core, r))
    ring.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: b200sac_soft_update on every family and replica
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("tau", [0.0, 0.005, 0.37, 1.0])
@pytest.mark.parametrize("name", ["chained_ll", "vs400_tc", "mtsac_t10", "care_m", "care_o"])
def test_soft_update_is_exact(cuda, name, tau):
    """Both critics with `tau`; the CARE target state encoder with the replica's tau_se, except at tau = 1 -- the hard
    copy of every target, tse included."""
    core, spec, care = _handle(name, R=3, rows=ROWS)
    for r in range(3):
        _plant_negative_zeros(core, r, per_tensor=16)
    before = [export(core, r) for r in range(3)]
    core.soft_update(tau)
    flipped = 0
    for r in range(3):
        after = export(core, r)
        rates = {"tau": tau, "tau_se": tau if tau == 1.0 else ROWS[r]["tau_se"]}
        check_targets(core, before[r], after, rates, True, f"{name} soft_update({tau}) replica {r}", _other_rates(core, r))
        for tname, lname, _k in target_pairs(core):
            off, rows, _c, _t, _o, pitch = core.table[tname]
            loff = core.table[lname][0]
            t_old, t_new = before[r][off:off + rows * pitch], after[off:off + rows * pitch]
            if tau == 1.0:
                assert np.array_equal(t_new, after[loff:loff + rows * pitch]), f"{name} replica {r}: {tname} is not a copy"
            flipped += int(((_bits(t_old) == 0x80000000) & (_bits(t_new) == 0)).sum())
    if tau == 0.0:
        assert flipped > 0, "no planted -0.0 target met a positive local: the tau = 0 edge was not exercised"
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: Learner.soft_update(local_critic_k, target_critic_k, tau) updates that pair only
# ---------------------------------------------------------------------------------------------------------------------
def _scramble_targets(core, seed):
    g = torch.Generator().manual_seed(seed)
    named = core.get_named()
    for k in named:
        if "_target." in k:
            named[k] = named[k] + 0.05 * torch.randn(named[k].shape, generator=g)
    core.set_named(named)


@pytest.mark.parametrize("family", ["LL", "VS"])
def test_learner_soft_update_moves_only_its_pair(cuda, tmp_path, monkeypatch, family):
    monkeypatch.chdir(tmp_path)
    lrn = _learner(family, tmp_path)
    core = lrn.core
    try:
        _scramble_targets(core, 1)
        tau = 0.3
        s0 = export(core)
        lrn.soft_update(lrn.local_critic_1, lrn.target_critic_1, tau)
        s1 = export(core)
        lrn.soft_update(lrn.local_critic_2, lrn.target_critic_2, tau)
        s2 = export(core)
        for i, (a, b, k) in enumerate(((s0, s1, 1), (s1, s2, 2))):
            for tname, lname, _key in target_pairs(core):
                off, rows, _c, _t, _o, pitch = core.table[tname]
                loff, n = core.table[lname][0], rows * pitch
                mine = tname.startswith(f"q{k}_target.")
                want = polyak(b[loff:loff + n], a[off:off + n], tau) if mine else a[off:off + n]
                assert np.array_equal(_bits(b[off:off + n]), _bits(want)), \
                    f"{family}: soft_update(local_critic_{k}, target_critic_{k}) {'wrong on' if mine else 'changed'} {tname}"
            assert np.array_equal(_bits(a[:core.trainable_floats]), _bits(b[:core.trainable_floats])), "a local changed"
        # the two pair calls compose to one update of both critics
        core.import_arena(torch.from_numpy(s0))
        core.soft_update(tau)
        assert np.array_equal(_bits(export(core)), _bits(s2)), "pair calls != one b200sac_soft_update"
        # run()'s order with tau = 1: exact copies
        core.import_arena(torch.from_numpy(s0))
        lrn.soft_update(lrn.local_critic_1, lrn.target_critic_1, 1.0)
        lrn.soft_update(lrn.local_critic_2, lrn.target_critic_2, 1.0)
        got = core.get_named()
        for tname, lname, _key in target_pairs(core):
            assert torch.equal(got[tname], got[lname]), f"{family}: {tname} is not a copy of {lname} after tau = 1"
        # (None, None) keeps the whole-critic update; any other pair is refused and changes nothing
        core.import_arena(torch.from_numpy(s0))
        lrn.soft_update(None, None, tau)
        assert np.array_equal(_bits(export(core)), _bits(s2))
        for bad in ((lrn.local_critic_1, lrn.target_critic_2), (lrn.target_critic_1, lrn.local_critic_1),
                    (lrn.actor, lrn.target_critic_1), (lrn.local_critic_2, None)):
            with pytest.raises(ValueError):
                lrn.soft_update(*bad, tau)
        assert np.array_equal(_bits(export(core)), _bits(s2))
    finally:
        lrn.memory.stop()
