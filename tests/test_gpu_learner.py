"""GPU: the reference-shaped Learner / ReplayBuffer surface (drop-in boundary)."""
import json
import os
import pickle

import pytest
import torch

import redis_stub
from _golden import Case, REL, rel_l2, rel_scalar
from _harness import LL_CFG, cuda

pytestmark = pytest.mark.gpu


def _ll_learner(tmp_path, **kw):
    from distributed_sac_b200.learner import Learner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(LL_CFG))
    os.chdir(tmp_path)
    return Learner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)), **kw)


def test_ll_learner_matches_fixture_through_reference_api(cuda, tmp_path):
    """Load the fixture through load_state_dict-style handles with the REFERENCE key names, run
    update_SAC() on the fixture minibatches, compare losses and the actor blob players would pull."""
    from distributed_sac_b200 import _lib, names
    c = Case("ll_ckpt_s3")
    lrn = _ll_learner(tmp_path)
    inv = lambda km, src: {ref: src[canon] for ref, canon in km.items()}
    lrn.actor.load_state_dict(inv(names.actor_key_map("LL", 3), c.p_in))
    lrn.local_critic_1.load_state_dict(inv(names.critic_key_map("LL", 3, 1), c.p_in))
    lrn.local_critic_2.load_state_dict(inv(names.critic_key_map("LL", 3, 2), c.p_in))
    lrn.target_critic_1.load_state_dict(inv(names.critic_key_map("LL", 3, 1, True), c.p_in))
    lrn.target_critic_2.load_state_dict(inv(names.critic_key_map("LL", 3, 2, True), c.p_in))
    lrn.core.set_named({"log_alpha": c.p_in["log_alpha"]}, strict=False)
    lrn.core.set_named(c.m_in, _lib.ADAM_M)
    lrn.core.set_named(c.v_in, _lib.ADAM_V)
    lrn.core.set_steps(c.step_in)
    for i in range(c.n_steps):
        s, a, r, s2, d = c.step_batch(i)
        dev = (i % 2 == 0)       # alternate device / host minibatches: both entry points
        mv = (lambda t: t.cuda()) if dev else (lambda t: t)
        cl, al = lrn.update_SAC(mv(s), mv(a), mv(r), mv(s2), mv(d), None, eps_next=mv(c.eps_next[i]), eps_cur=mv(c.eps_cur[i]))
        assert rel_scalar(cl, c.losses[i, 0]) <= REL and rel_scalar(al, c.losses[i, 1]) <= REL
    blob = pickle.loads(pickle.dumps(lrn.get_parameters()))       # what run() publishes to players
    assert set(blob) == {"actor"}
    km = names.actor_key_map("LL", 3)
    assert set(blob["actor"]) == set(km)
    for ref, canon in km.items():
        assert blob["actor"][ref].shape == c.p_out[canon].shape
        assert rel_l2(blob["actor"][ref], c.p_out[canon]) <= REL
    lrn.memory.stop()


def test_checkpoint_round_trip_in_reference_format(cuda, tmp_path):
    lrn = _ll_learner(tmp_path, seed=3)
    lrn.memory.ring.fill_synthetic(20000, seed=1)
    for _ in range(5):
        cl, al = lrn.update()
        assert cl == cl and al == al
    path = lrn.save_checkpoint(15)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert {"episode_idx", "total_step", "local_critic_1", "local_critic_2", "critic_optimizer", "target_critic_1",
            "target_critic_2", "actor", "actor_optimizer", "log_alpha", "log_alpha_optimizer", "alpha"} <= set(ck)
    assert set(ck["local_critic_1"]) == {"first_layer.weight", "first_layer.bias", "layer_module.0.weight",
                                         "layer_module.0.bias", "layer_module.1.weight", "layer_module.1.bias"}
    assert len(ck["critic_optimizer"]["state"]) == 12 and int(ck["critic_optimizer"]["state"][0]["step"]) == 5
    # a plain torch Adam accepts the saved optimizer state (the format players / tools rely on)
    ps = [torch.nn.Parameter(torch.zeros_like(ck["critic_optimizer"]["state"][i]["exp_avg"])) for i in range(12)]
    torch.optim.Adam(ps, lr=3e-4).load_state_dict(ck["critic_optimizer"])
    before = lrn.core.export_arena()
    lrn2 = _ll_learner(tmp_path, seed=9, checkpoint_path=path)
    assert torch.equal(lrn2.core.export_arena(), before)
    assert lrn2.core.get_steps() == (5, 5, 5)
    s, a, r, s2, d = lrn.memory.sample()
    assert s.is_cuda and s.shape == (256, 8) and a.shape == (256, 2) and r.shape == (256, 1) and d.shape == (256, 1)
    g = torch.Generator().manual_seed(0)
    e1, e2 = torch.randn(256, 2, generator=g), torch.randn(256, 2, generator=g)
    assert lrn.update_SAC(s, a, r, s2, d, None, eps_next=e1.cuda(), eps_cur=e2.cuda()) == \
        lrn2.update_SAC(s, a, r, s2, d, None, eps_next=e1.cuda(), eps_cur=e2.cuda())
    lrn.memory.stop()
    lrn2.memory.stop()


def test_run_loop_with_redis_stub(cuda, tmp_path):
    """Learner.run(): players push pickled tuples to the 'sample' list, the ReplayBuffer thread drains
    them, the learner publishes 'parameters' / 'update_iteration' and loss lists (LL/learner.py:278-316)."""
    import numpy as np
    lrn = _ll_learner(tmp_path, seed=1)
    lrn.write_mode = True
    lrn.start_memory_len = 1200
    rng = np.random.default_rng(0)
    for _ in range(1500):      # tuple layout of LL/player.py:115-122
        tup = (rng.standard_normal(8), rng.uniform(-1, 1, 2).astype(np.float32), float(rng.standard_normal()),
               rng.standard_normal(8), bool(rng.random() < 0.01))
        lrn.server.rpush("sample", pickle.dumps(tup))
    n = lrn.run(max_updates=7)
    assert n == 7 and len(lrn.memory) == 1500
    assert pickle.loads(lrn.server.get("update_iteration")) == 18          # update_delay = 3
    params = pickle.loads(lrn.server.get("parameters"))
    assert params["actor"]["mu_log_std_layer.weight"].shape == (4, 256)
    assert lrn.server.llen("critic_loss") == 7 and lrn.server.llen("alpha") == 7
    # the last published blob (assembled on the device, b200sac_blob_*) is the actor after the last update, and the logged
    # temperature is the one of the same snapshot
    final = lrn._module_state_dict("actor")
    assert all(torch.equal(params["actor"][k], final[k]) for k in final)
    it, alphas = pickle.loads(lrn.server.pipeline().lrange("alpha", 6, 6).execute()[0][0])
    assert it == 18 and np.allclose(alphas, lrn.log_alpha.exp().numpy(), rtol=1e-6)
    lrn.memory.stop()


def test_mtsac_learner_action_bound_sets_the_action_scale(cuda, tmp_path):
    """MTSACLearner reads action_bound from its cfg's actor block (MS/learner.py): [-2, 2] gives a core with action scale 2,
    and acting in every mode stays within the bound and uses it (a head that ignored the scale would stay within 1)."""
    from distributed_sac_b200.learner import MTSACLearner
    T = 4
    cfg = {"device": "cuda", "buffer_size": 4096, "reward_scale": 1, "batch_size": 64, "gamma": 0.99, "tau": 0.005,
           "log_alpha": 0, "start_memory_len": 1000, "print_period_learner": 10, "update_delay": 1, "num_tasks": T,
           "actor": {"lr_actor": 3e-4, "state_dim": 12, "action_dim": 3, "action_bound": [-2.0, 2.0], "actor_hidden_dim": [64, 64]},
           "critic": {"lr_critic": 3e-4, "critic_hidden_dim": [64, 64]}}
    p = tmp_path / "ms.json"
    p.write_text(json.dumps(cfg))
    lrn = MTSACLearner(None, [f"t{i}" for i in range(T)], str(p), write_mode=False, replay_where="device",
                       server=redis_stub.StrictRedis(host=str(tmp_path) + "ms"))
    try:
        assert lrn.core.cfg.action_scale == 2.0
        g = torch.Generator().manual_seed(0)
        obs = torch.cat([3 * torch.randn(128, 12, generator=g), torch.eye(T)[torch.arange(128) % T]], 1)
        for stochastic in (True, False):
            a = lrn.act_batch(obs, stochastic=stochastic)
            assert a.shape == (128, 3) and torch.isfinite(a).all()
            assert float(a.abs().max()) <= 2.0 and float(a.abs().max()) > 1.0, (stochastic, float(a.abs().max()))
        lrn.memory.ring.fill_synthetic(4096, seed=1)
        assert all(x == x for x in lrn.update())
    finally:
        lrn.memory.stop()


@pytest.mark.parametrize("modified", [True, False], ids=["CARE(M)", "CARE(O)"])
def test_care_learner_surface(cuda, tmp_path, modified):
    """CARELearner: cfg 'encoder' block + metadata JSONs as in MT10_Distributed_CARE_cfg.json; published blob has the
    reference's keys/shapes (Player loads context_encoder + actor state_dicts, C10/player.py:82-93)."""
    import numpy as np
    from distributed_sac_b200.learner import CARELearner
    names_ = [f"task-{i}" for i in range(10)]
    rng = np.random.default_rng(0)
    emb = {n: rng.standard_normal(768).round(4).tolist() for n in names_}
    (tmp_path / "emb.json").write_text(json.dumps(emb))
    (tmp_path / "names.json").write_text(json.dumps(names_))
    cfg = {"use_modified_care": modified, "num_tasks": 10, "device": "cuda", "buffer_size": 40000, "reward_scale": 1,
           "batch_size": 160, "log_alpha": 0, "tau": 0.005, "update_delay": 6, "random_step": 5000, "start_memory_len": 5000,
           "print_period_player": 2, "print_period_learner": 10, "gamma": 0.99, "max_episode_time": 500,
           "actor": {"state_dim": 39, "action_dim": 4, "action_bound": [-1.0, 1.0], "lr_actor": 3e-4, "actor_hidden_dim": [64, 64, 64]},
           "critic": {"state_dim": 39, "action_dim": 4, "lr_critic": 3e-4, "critic_hidden_dim": [64, 64, 64]},
           "encoder": {"state_dim": 39, "pretrained_embedding_json_path": str(tmp_path / "emb.json"),
                       "task_name_json_path": str(tmp_path / "names.json"), "hidden_dims_contextEnc": [50, 50],
                       "embedding_dim_contextEnc": 50, "output_dim_contextEnc": 50, "RoBERTa_embedding_dim": 768,
                       "lr_contextEnc": 3e-4, "hidden_dims_mixtureEnc": [50], "output_dim_mixtureEnc": 50, "num_encoders": 6,
                       "num_tasks": 10, "state_encoder_tau": 0.05}}
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(cfg))
    os.chdir(tmp_path)
    lrn = CARELearner(None, names_, str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "c"))
    lrn.memory.ring.fill_synthetic(40000, seed=1)
    for _ in range(4):
        cl, al, ent = lrn.update()
        assert cl == cl and al == al and ent == ent
    blob = pickle.loads(pickle.dumps(lrn.get_parameters()))
    assert set(blob) == {"context_encoder", "actor"}
    E = blob["context_encoder"]["embedding.0.weight"]
    assert E.shape == (10, 768) and torch.allclose(E, torch.tensor([emb[n] for n in names_]))
    a = blob["actor"]
    assert a["state_encoder.mixture_encoders.mixtureEncoders.0.W"].shape == (6, 39, 50)
    assert a["state_encoder.mixture_encoders.mixtureEncoders.0.b"].shape == (6, 1, 50)
    assert a["state_encoder.mixture_encoders.mixtureEncoders.2.W"].shape == (6, 50, 50)
    assert a["state_encoder.trunk.0.weight"].shape == (50, 768 if modified else 50) and a["state_encoder.trunk.2.weight"].shape == (6, 50)
    if modified:
        assert a["state_encoder.mlp_context.4.weight"].shape == (50, 50)
    else:       # CARE(O): trainable context encoder published to the players (C10/player.py:82-93)
        ce = blob["context_encoder"]
        assert "state_encoder.mlp_context.0.weight" not in a
        assert ce["embedding.2.0.weight"].shape == (100, 768) and ce["embedding.2.2.weight"].shape == (50, 100)
        assert ce["mlp.0.weight"].shape == (50, 50) and ce["mlp.4.bias"].shape == (50,)
    assert a["mu_log_std_layer.0.weight"].shape == (64, 100) and a["mu_log_std_layer.6.weight"].shape == (8, 64)
    path = lrn.save_checkpoint(24)
    ck = torch.load(path, map_location="cpu", weights_only=False)
    assert "state_encoder.trunk.0.weight" in ck["local_critic"] and "Q_function_2.6.bias" in ck["target_critic"]
    assert len(ck["critic_optimizer"]["state"]) == (14 if modified else 8) + 16 and len(ck["actor_optimizer"]["state"]) == 8
    # MTSAC / CARE checkpoints carry 'update_iteration' (C10/learner.py:180,202), and the context-encoder optimizer is
    # Adam(context_encoder.parameters()): parameter 0 = the frozen embedding (never any state), CARE(M) has nothing else
    assert ck["update_iteration"] == 24 and "episode_idx" not in ck
    ceo = ck["context_encoder_optimizer"]
    if modified:
        assert ceo["state"] == {} and ceo["param_groups"][0]["params"] == [0]
    else:
        assert sorted(ceo["state"]) == list(range(1, 11)) and int(ceo["state"][1]["step"]) == 4
        assert ceo["param_groups"][0]["params"] == list(range(11))
        assert ceo["state"][1]["exp_avg"].shape == (100, 768) and ceo["state"][10]["exp_avg"].shape == (50,)
    # the bytes run() publishes, once unpickled == every published module read out of the whole arena
    pub = pickle.loads(lrn.parameters_blob(blocking=True))
    assert set(pub) == set(lrn._published)
    for net in pub:
        full = lrn._module_state_dict(net)
        assert set(pub[net]) == set(full)
        for k in full:
            assert pub[net][k].dtype == torch.float32 and torch.equal(pub[net][k], full[k]), (net, k)
    before = lrn.core.export_arena()
    lrn2 = CARELearner(None, names_, str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "d"),
                       seed=5, checkpoint_path=path)
    assert torch.equal(lrn2.core.export_arena(), before)
    lrn.memory.stop()
    lrn2.memory.stop()


def test_published_blob_is_consistent_and_async(cuda, tmp_path):
    """get_parameters() and the published blob (b200sac_blob_*): (1) bit-identical to the full-arena export; (2) a blob
    begun after step k and collected after further steps were enqueued is the state after step k, not a torn
    or later one (it is what an unmodified Player would load, LL/player.py:75-85)."""
    lrn = _ll_learner(tmp_path, seed=11)
    twin = _ll_learner(tmp_path, seed=11)
    for l in (lrn, twin):
        l.memory.ring.fill_synthetic(20000, seed=2)
    for _ in range(3):
        lrn.update(); twin.update()
    full = lrn._module_state_dict("actor")                       # slow path: whole arena D2H
    blob = lrn.get_parameters()["actor"]
    assert set(blob) == set(full) and all(torch.equal(blob[k], full[k]) for k in full)
    fast = pickle.loads(lrn.parameters_blob(blocking=True))["actor"]      # template-patched pickle stream (run() publishes this)
    assert set(fast) == set(full) and all(torch.equal(fast[k], full[k]) and fast[k].is_contiguous() for k in full)
    assert torch.equal(lrn.log_alpha, lrn.core.get_named()["log_alpha"])          # small-range read == arena export
    lrn.core.blob_begin()                                        # the device-assembled blob after step 3 ...
    lrn.core.step_sampled(lrn.memory.ring, 40)                   # ... while 40 more steps are enqueued behind it
    blob3, extra3 = lrn.core.blob_wait()
    snap_b = pickle.loads(blob3)["actor"]
    assert all(torch.equal(snap_b[k], full[k]) for k in full)
    twin.core.step_sampled(twin.memory.ring, 40)                 # same seed, same ring: replicas stay bit-identical
    after, ref = lrn.get_parameters()["actor"], twin.get_parameters()["actor"]
    assert all(torch.equal(after[k], ref[k]) for k in ref)
    assert not torch.equal(after["mu_log_std_layer.weight"], full["mu_log_std_layer.weight"])
    lrn.memory.stop(); twin.memory.stop()
