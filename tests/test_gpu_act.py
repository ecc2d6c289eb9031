"""GPU: batched policy inference (b200sac_act) against the oracle's Actor.get_action restatement.

Reference: Actor.forward / get_action, LunarLander_Distributed_SAC/src/model.py:38-48,67-82 (MT: MT10_Distributed_MTSAC/src/model.py:35-73).
Tolerance: REL = 1e-4 on the action tensor (same bar as the step's `a` intermediates)."""
import pytest
import torch

import sac_port as sp
from _golden import Case, REL, core_config, rel_l2
from _harness import cuda

pytestmark = pytest.mark.gpu


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("name", ["ll_ckpt_s3", "ms_small_s5"])
def test_act_matches_oracle_policy(cuda, name, precision):
    from distributed_sac_b200.core import SacCore
    c = Case(name)
    core = SacCore(core_config(c.spec, precision=precision), 0, seed=0)
    core.set_named(c.p_in)
    s = c.step_batch(0)[0]
    B, A = s.shape[0], c.spec.act_dim
    g = torch.Generator().manual_seed(3)
    obs = torch.cat([s, c.step_batch(1)[3]])[: 2 * B]                     # 2B rows: the maximum one call takes
    eps = torch.randn(obs.shape[0], A, generator=g)
    ref, _, _ = sp.policy_sample(c.spec, c.p_in, obs, eps)
    assert rel_l2(core.act(obs, eps=eps), ref) <= REL
    det, _, _ = sp.policy_sample(c.spec, c.p_in, obs[:7], torch.zeros(7, A))      # k * tanh(mu), ragged row count
    assert rel_l2(core.act(obs[:7].cuda(), stochastic=False), det) <= REL            # device-resident observations too
    a1, a2 = core.act(obs[:64]), core.act(obs[:64])                                  # fresh noise per call
    assert not torch.equal(a1, a2) and a1.abs().max() <= c.spec.action_scale + 1e-6
    # acting does not disturb training: the fixture's first step still matches the reference afterwards
    core.step(*c.step_batch(0), c.eps_next[0], c.eps_cur[0])
    for k, refv in c.i0.items():
        assert rel_l2(core.debug(k).reshape(refv.shape), refv) <= REL, k
    with pytest.raises(RuntimeError):
        core.act(torch.zeros(2 * B + 1, obs.shape[1]))
    core.close()


def test_learner_act_batch_surface(cuda, tmp_path):
    import json, os
    import redis_stub
    from distributed_sac_b200.learner import Learner
    cfg = {"num_tasks": 10, "device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 256, "gamma": 0.99,
           "lr_actor": 3e-4, "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "num_learn": 1, "num_time_step": 1,
           "random_step": 5000, "start_memory_len": 5000}
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(cfg))
    os.chdir(tmp_path)
    lrn = Learner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)))
    obs = torch.randn(100, 8)
    acts = lrn.act_batch(obs.numpy(), stochastic=False)
    # the LunarLander actor's deterministic action is k * mu WITHOUT tanh (LunarLander_Distributed_SAC/src/model.py:78-80)
    mu = sp.mlp(lrn.core.get_named(), "actor", obs)[:, :2]
    assert acts.shape == (100, 2) and rel_l2(acts, mu) <= REL
    sto = lrn.act_batch(obs.numpy(), stochastic=True)
    assert sto.abs().max() <= 1.0 and not torch.equal(sto, acts)
    lrn.memory.stop()


@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("name", ["care_small_s4", "care_o_small_s4", "care_mt1_small_s3"], ids=["CARE(M)", "CARE(O)", "MT1-CARE"])
def test_act_care_matches_oracle_policy(cuda, name, precision):
    """b200sac_act on CARE handles = the player's inference path: z = context_encoder(mtobs), then the actor over its
    (tied) state encoder (MT10_Distributed_CARE/src/player.py:199-209, model.py:90-114), vs oracle/care_port.py."""
    import care_port as cp
    from _golden import CareCase, care_core_config
    from distributed_sac_b200.core import SacCore
    c = CareCase(name)
    core = SacCore(care_core_config(c.spec, precision=precision), 0, seed=0)
    core.set_named(c.p_in)
    port = cp.CarePortLearner(c.spec, c.p_in)
    B, A = c.spec.batch, c.spec.act_dim
    obs = torch.cat([c.step_batch(0)[0][: B // 2], c.step_batch(1)[3][: B - B // 2]])      # B rows of mixed tasks
    g = torch.Generator().manual_seed(4)
    eps = torch.randn(B, A, generator=g)
    with torch.no_grad():
        tid = torch.argmax(obs[:, -c.spec.num_tasks:], dim=1)
        z = cp.context_encode(c.spec, port.p, tid)
        ref, _, _ = port._policy("ase", z, obs, eps, False)
        det, _, _ = port._policy("ase", z[:9], obs[:9], torch.zeros(9, A), False)
    assert rel_l2(core.act(obs, eps=eps), ref) <= REL
    assert rel_l2(core.act(obs[:9].cuda(), stochastic=False), det) <= REL
    # acting does not disturb training: the fixture's first step still matches the reference afterwards
    core.step(*c.step_batch(0), c.eps_next[0], c.eps_cur[0])
    for k, refv in c.i0.items():
        assert rel_l2(core.debug(k).reshape(refv.shape), refv) <= REL, k
    with pytest.raises(RuntimeError):
        core.act(torch.zeros(B + 1, obs.shape[1]))
    core.close()
