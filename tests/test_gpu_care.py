"""GPU: the CARE(M) step (context embedding + mixture-of-encoders state encoders) against the fixture
generated from the real MT10_Distributed_CARE learner and against the CPU oracle at full size."""
import pytest
import torch

import care_port as cp
from _golden import CareCase, REL, care_core_config, check_port_state, check_state, kink_checked_step, rel_l2, rel_scalar
from _harness import cuda

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("name", ["care_small_s4", "care_o_small_s4", "care_mt1_small_s3"], ids=["CARE(M)", "CARE(O)", "MT1-CARE"])
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
def test_care_step_matches_reference_fixture(cuda, precision, name):
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import SacCore
    c = CareCase(name)
    core = SacCore(care_core_config(c.spec, precision=precision), 0, seed=0)
    core.set_named(c.p_in)
    for i in range(c.n_steps):
        core.step(*c.step_batch(i), c.eps_next[i], c.eps_cur[i])
        if i == 0:
            for k, ref in c.i0.items():
                got = core.debug(k).reshape(ref.shape)
                assert rel_l2(got, ref) <= REL, (k, rel_l2(got, ref))
        L = core.read_losses(1)[0, 0]
        assert rel_scalar(float(L[0]), c.losses[i, 0]) <= REL, ("critic_loss", i, float(L[0]), c.losses[i, 0])
        assert rel_scalar(float(L[1]), c.losses[i, 1]) <= REL, ("actor_loss", i, float(L[1]), c.losses[i, 1])
        assert rel_scalar(float(L[3]), c.losses[i, 2]) <= REL, ("entropy", i)
    check_state(c, core.get_named(_lib.PARAMS), core.get_named(_lib.ADAM_M), core.get_named(_lib.ADAM_V),
                core.get_steps(), what="CUDA CARE state")
    core.close()


@pytest.mark.parametrize("modified", [True, False], ids=["CARE(M)", "CARE(O)"])
def test_care_full_size_matches_port(cuda, modified):
    """BASELINE.json config 5 shape: 39+10 obs, K=6 encoders, 768-d context, 400^3 MLPs, batch 1280 -- everything at
    1e-4 with the ReLU kinks proven (tests/_golden.py::kink_checked_step; masks of the consumer MLPs and of the
    mixture-encoder hidden layers are forced, the 10-row per-task MLPs keep the oracle's own)."""
    from distributed_sac_b200.core import SacCore
    spec = cp.CareSpec(modified=modified, weighted_loss=modified)
    p = cp.init_params(spec, seed=2)
    port = cp.CarePortLearner(spec, p)
    core = SacCore(care_core_config(spec, precision=1), 0, seed=0)
    gen = torch.Generator().manual_seed(5)
    for i in range(2):
        b = cp.synthetic_batch(spec, seed=50 + i)
        e1 = torch.randn(spec.batch, spec.act_dim, generator=gen)
        e2 = torch.randn(spec.batch, spec.act_dim, generator=gen)
        o, flips = kink_checked_step(core, port, spec, b, e1, e2, care=True)
        L = core.read_losses(1)[0, 0]
        assert rel_scalar(float(L[0]), o["critic_loss"]) <= REL, (i, float(L[0]), o["critic_loss"])
        assert rel_scalar(float(L[1]), o["actor_loss"]) <= REL, (i, float(L[1]), o["actor_loss"])
        assert rel_scalar(float(L[3]), o["entropy"]) <= REL
        check_port_state(core, port)
    core.close()
