"""CPU: the oracle ports and the host-side wire formats against data WRITTEN BY THE UNMODIFIED REFERENCE and stored under
tests/golden/ (oracle/gen_golden.py, oracle/gen_checkpoints.py generate it from a reference checkout; nothing here needs one):

* oracle/sac_port.py reproduces the reference learner's update() step for step at the bound the port keeps against the
  live reference (1e-5 on losses and parameters): the stored fixtures are the reference's own outputs for the stored
  parameters, minibatches and noise;
* the bytes Learner.run() publishes (Learner.parameters_blob: a pickle stream built once whose float payloads the library
  gathers from the arena) carry exactly the state_dict a reference Actor wrote -- same keys in the same order, shapes,
  dtypes and values -- which is what Player.pull_parameters' strict load_state_dict needs (LL/player.py:75-85);
* the reference-written checkpoints have the key sets the reference's load_checkpoint() reads, and their module
  state_dicts use exactly the keys the drop-in learner maps (distributed_sac_b200/names.py)."""
import pickle

import numpy as np
import pytest
import torch

import sac_port as sp
from _golden import Case, golden_file, rel_l2, rel_scalar


@pytest.mark.parametrize("family,case", [("LL", "ll_xavier_s2"), ("MS", "ms_small_s5")])
def test_port_follows_the_live_reference(family, case):
    c = Case(case)
    assert c.family == family
    port = sp.PortLearner(c.spec, c.p_in, {"m": c.m_in, "v": c.v_in, "step": tuple(c.step_in)})
    for i in range(c.n_steps):
        o = port.update_SAC(*c.step_batch(i), eps_next=c.eps_next[i], eps_cur=c.eps_cur[i])
        res = c.losses[i]
        assert rel_scalar(o["critic_loss"], res[0]) <= 1e-5 and rel_scalar(o["actor_loss"], res[1]) <= 1e-5, (i, o, res)
    got = port.params()
    for k, p in c.p_out.items():
        if k == "log_alpha":
            assert (got[k].double() - p.double()).abs().max().item() <= 1e-6
        else:
            assert rel_l2(got[k], p) <= 1e-5, (k, rel_l2(got[k], p))


def test_published_blob_loads_into_the_reference_actor(tmp_path):
    """parameters_blob() is host logic: exercised here with a stand-in core whose arena holds the actor state_dict the
    reference's own Actor wrote into a checkpoint; the unpickled blob must be that state_dict exactly (what a strict
    load_state_dict into a reference Actor requires)."""
    from distributed_sac_b200 import names
    from distributed_sac_b200.learner import _BaseLearner
    ck = torch.load(golden_file("ref_ckpt_ll_small.tar", tmp_path), map_location="cpu", weights_only=False)
    sd = ck["actor"]
    km = names.actor_key_map("LL", 3)
    assert list(km) == list(sd)

    # stand-in core: the arena of a LunarLander learner filled with the reference Actor's state; the device gather of
    # b200sac_blob_* is emulated on the CPU (tests/_harness.py::BlobStubLib)
    import distributed_sac_b200.core as core_mod
    from distributed_sac_b200.core import CoreConfig, SacCore, layout
    from _harness import BlobStubLib
    cfg = CoreConfig(batch=64)
    table, arena, _tr = layout(cfg)
    flat = np.zeros(arena, np.float32)
    core = object.__new__(SacCore)
    core.lib, core._h, core.cfg, core.table = BlobStubLib(flat), None, cfg, table
    for ref, canon in km.items():
        off, rows, cols, _t, _o, pitch = table[canon]
        flat[off:off + rows * pitch].reshape(rows, pitch)[:, :cols] = sd[ref].detach().numpy().reshape(rows, cols)
    shim = _BaseLearner.__new__(_BaseLearner)
    shim.core = core
    shim._key_map = lambda net: km
    real_stream = core_mod._stream
    core_mod._stream = lambda: None
    try:
        blob = shim.parameters_blob()
    finally:
        core_mod._stream = real_stream
    params = pickle.loads(blob)                                   # Player.pull_parameters: _pickle.loads(server.get('parameters'))
    assert list(params) == ["actor"] and list(params["actor"]) == list(sd)
    for k, v in sd.items():
        got = params["actor"][k]
        assert isinstance(got, torch.Tensor) and got.shape == v.shape and got.dtype == v.dtype, k
        assert torch.equal(got, v), k


def test_reference_load_checkpoint_reads_the_keys_we_write(tmp_path):
    """Key sets of the reference-written fixtures == what each reference load_checkpoint() indexes (LL/learner.py:165-182,
    MS:176-190, C10:200-217); tests/test_gpu_checkpoint.py proves the drop-in learner writes exactly these trees."""
    from distributed_sac_b200 import names
    want = {
        "ref_ckpt_ll_small": {"episode_idx", "total_step", "local_critic_1", "local_critic_2", "critic_optimizer", "target_critic_1",
                              "target_critic_2", "actor", "actor_optimizer", "log_alpha", "log_alpha_optimizer", "alpha"},
        "ref_ckpt_ms_small": {"update_iteration", "total_step", "local_critic", "critic_optimizer", "target_critic", "actor",
                              "actor_optimizer", "log_alpha", "log_alpha_optimizer", "alpha"},
        "ref_ckpt_c10m_small": {"update_iteration", "total_step", "context_encoder", "context_encoder_optimizer", "local_critic",
                                "critic_optimizer", "target_critic", "actor", "actor_optimizer", "log_alpha", "log_alpha_optimizer", "alpha"},
    }
    for name, keys in want.items():
        ck = torch.load(golden_file(name + ".tar", tmp_path), map_location="cpu", weights_only=False)
        assert set(ck) == keys, (name, set(ck) ^ keys)
    # the module state_dicts of the LunarLander checkpoint use exactly the keys the drop-in learner maps, and its critic
    # optimizer state is the reference's after the two updates the fixture ran
    ck = torch.load(golden_file("ref_ckpt_ll_small.tar", tmp_path), map_location="cpu", weights_only=False)
    assert list(ck["actor"]) == list(names.actor_key_map("LL", 3))
    for which in (1, 2):
        assert list(ck[f"local_critic_{which}"]) == list(names.critic_key_map("LL", 3, which))
        assert list(ck[f"target_critic_{which}"]) == list(names.critic_key_map("LL", 3, which, True))
    assert int(ck["critic_optimizer"]["state"][0]["step"]) == 2
