"""GPU: the CUDA step against the full-size fixtures of the UNMODIFIED reference (BASELINE.json configs 3-5 at their
configured shapes and a 100-step LunarLander chain; oracle/gen_golden.py FULL_CASES, pinned to the port on CPU by
tests/test_oracle_fullsize.py).

The CUDA learner runs the whole chain on its own (no re-synchronisation).  Checked against the reference fixture,
strictly at 1e-4: the first step's forward intermediates and the losses of every step up to the first proven ReLU kink
(after a kink two correct fp32 chains separate slowly; from there on the losses are held to the port that follows the
same masks).  The gradient-derived state is checked strictly at 1e-4 too, with the kinks proven instead of
budgeted: a port learner follows the same chain with the masks the CUDA step used forced in (tests/_golden.py), every
forced bit that differs from the port's own must sit on a numerically-zero pre-activation, and the final CUDA state must
equal that port's state; when no bit differed at all, the CUDA state must equal the reference's summary directly."""
import math

import pytest

import sac_port as sp
from _golden import (check_forced, FULL_CARE_CASES, FULL_CASES, REL, FullCase, care_core_config, check_port_state, core_config,
                     cuda_relu_masks, rel_l2, rel_scalar)
from _harness import cuda

pytestmark = pytest.mark.gpu


def _cases():
    out = []
    for name in FULL_CASES + FULL_CARE_CASES:
        for precision in (0, 1):
            if name in FULL_CARE_CASES and precision == 0:
                continue          # (CARE at B = 1280 in exact-fp32 FFMA is covered by the small fixtures; 3xTF32 is its production mode)
            out.append(pytest.param(name, precision, id=f"{name}-{'fp32' if precision == 0 else 'tc3xtf32'}"))
    return out


@pytest.mark.parametrize("name,precision", _cases())
def test_chain_matches_reference_fixture_at_full_size(cuda, name, precision):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    c = FullCase(name)
    cfg = care_core_config(c.spec, precision=precision) if c.care else core_config(c.spec, precision=precision)
    core = SacCore(cfg, 0, seed=0)
    core.set_named(c.params)
    port = c.make_port()
    total_flips, direct_steps = 0, 0
    for i in range(c.n_steps):
        core.step(*c.batches[i], c.eps_next[i], c.eps_cur[i])
        if i == 0:
            for k, ref in c.i0.items():
                got = core.debug(k).reshape(ref.shape)
                assert rel_l2(got, ref) <= REL, (k, rel_l2(got, ref))
        L = core.read_losses(1)[0, 0]
        if total_flips == 0:            # no kink so far: the reference's own losses, strictly
            assert rel_scalar(float(L[0]), c.losses[i, 0]) <= REL, ("critic_loss", i, float(L[0]), c.losses[i, 0])
            assert rel_scalar(float(L[1]), c.losses[i, 1]) <= REL, ("actor_loss", i, float(L[1]), c.losses[i, 1])
            if not math.isnan(c.losses[i, 2]):
                assert rel_scalar(float(L[3]), c.losses[i, 2]) <= REL, ("entropy", i)
            direct_steps = i + 1
        # the same step in the port with the CUDA masks forced; differing bits must be kinks
        forced = cuda_relu_masks(core, c.spec, 0, c.care)
        with sp.ReluTape(forced) as tape:
            o = port.update_SAC(*c.batches[i], c.eps_next[i], c.eps_cur[i])
        # ... and with the same masks the two chains agree at every step (after a kink the trajectories of two correct
        # fp32 learners separate from the fixture's -- slowly, 1e-4 on the critic loss after ~95 LunarLander steps --
        # which is why the fixture comparison above stops at the first proven kink and this one never does)
        assert rel_scalar(float(L[0]), o["critic_loss"]) <= REL, ("critic_loss vs port with forced masks", i, float(L[0]), o["critic_loss"])
        assert rel_scalar(float(L[1]), o["actor_loss"]) <= REL, ("actor_loss vs port with forced masks", i, float(L[1]), o["actor_loss"])
        total_flips += sum(check_forced(tape, forced, f"step {i}: ").values())
    check_port_state(core, port)                       # strict 1e-4: CUDA chain == port chain with the same masks
    assert tuple(core.get_steps()) == tuple(int(x) for x in c.step_out)
    if total_flips == 0:                               # no kink anywhere in the chain: the reference's own numbers, directly
        c.check_summary("p_out", core.get_named(_lib.PARAMS), REL, "CUDA parameters")
        c.check_summary("m_out", core.get_named(_lib.ADAM_M), REL, "CUDA Adam m")
        c.check_summary("v_out", core.get_named(_lib.ADAM_V), REL, "CUDA Adam v")
    print(f"[kinks] {name} precision {precision}: {total_flips} mask bits differed over {c.n_steps} steps (all at numerically-zero "
          f"pre-activations); losses compared with the reference fixture directly for the first {direct_steps} steps")
    core.close()
