"""GPU: checkpoint interoperability with the reference (SURVEY.md 8(f) rank 3).

tests/golden/ref_ckpt_*.tar were WRITTEN BY THE UNMODIFIED REFERENCE's own save_checkpoint() (oracle/gen_checkpoints.py:
toy-sized learners after two update() steps; LunarLander at its hard-coded full size).  For every family:
  * the drop-in learner's load_checkpoint() accepts the file (LL/learner.py:165-182 is what the reference intends);
  * a checkpoint then saved by the drop-in learner has exactly the reference's structure -- top-level keys (incl.
    'episode_idx' vs 'update_iteration'), state_dict keys, shapes, dtypes, optimizer state indices (the frozen CARE
    embedding is parameter 0 of the context-encoder optimizer and has no state), param_groups -- and identical values,
    which is what makes it loadable by the reference's load_state_dict calls;
  * the next gradient step from the loaded state reproduces the reference's (losses and parameters to 1e-4)."""
import json
import math
import os

import pytest
import torch

import redis_stub
from _golden import REL, golden_file, load_npz, rel_l2, rel_scalar
from _harness import cuda

pytestmark = pytest.mark.gpu

CASES = ["ref_ckpt_ll_small", "ref_ckpt_vs_small", "ref_ckpt_ms_small", "ref_ckpt_c10m_small", "ref_ckpt_c10o_small"]


def _learner(variant, cfg_path, tmp_path, checkpoint):
    from distributed_sac_b200 import learner as L
    srv = redis_stub.StrictRedis(host=str(tmp_path) + variant)
    kw = dict(write_mode=False, server=srv, checkpoint_path=checkpoint, precision=0)
    if variant == "LL":
        return L.LunarLanderLearner(cfg_path, **kw)
    if variant == "VS":
        return L.VSACLearner(cfg_path, **kw)
    names = [f"task-{i}" for i in range(10)]
    return (L.CARELearner if variant == "C10" else L.MTSACLearner)(None, names, cfg_path, **kw)


def _same_tree(a, b, path=""):
    """identical nesting, keys, tensor shapes / dtypes and values"""
    if isinstance(b, dict):
        assert isinstance(a, dict) and set(a) == set(b), (path, sorted(map(str, set(a) ^ set(b))))
        for k in b:
            _same_tree(a[k], b[k], f"{path}/{k}")
    elif isinstance(b, (list, tuple)):
        assert len(a) == len(b), path
        for i, (x, y) in enumerate(zip(a, b)):
            _same_tree(x, y, f"{path}[{i}]")
    elif isinstance(b, torch.Tensor):
        assert isinstance(a, torch.Tensor) and a.shape == b.shape and a.dtype == b.dtype, (path, getattr(a, "shape", None), b.shape)
        assert torch.equal(a.detach().cpu(), b.detach().cpu()), (path, (a.detach().cpu().float() - b.detach().cpu().float()).abs().max())
    else:
        assert a == b, (path, a, b)


@pytest.mark.parametrize("name", CASES)
def test_reference_written_checkpoint_loads_saves_and_continues(cuda, tmp_path, monkeypatch, name):
    z = load_npz(name)
    tar = golden_file(name + ".tar", tmp_path)
    variant = str(z["variant"])
    cfg = json.loads(str(z["cfg"]))
    cfg["device"] = "cuda"
    cfg_path = tmp_path / "cfg.json"
    cfg_path.write_text(json.dumps(cfg))
    os.chdir(tmp_path)
    monkeypatch.setenv("B200SAC_ALLOW_RANDOM_EMBEDDING", "1")     # the RoBERTa table comes with the checkpoint, not from cfg/metadata
    ref = torch.load(tar, map_location="cpu", weights_only=False)
    lrn = _learner(variant, str(cfg_path), tmp_path, tar)
    assert lrn.total_step == 4321
    mine = torch.load(lrn.save_checkpoint(12), map_location="cpu", weights_only=False)
    _same_tree(mine, ref)
    # the next step from the loaded state == the reference's next step
    batch = [torch.from_numpy(z["batch/" + k]).cuda() for k in ("s", "a", "r", "s2", "d")]
    res = lrn.update_SAC(*batch, None, eps_next=torch.from_numpy(z["eps_next"]).cuda(), eps_cur=torch.from_numpy(z["eps_cur"]).cuda())
    want = z["losses"]
    assert rel_scalar(res[0], want[0]) <= REL and rel_scalar(res[1], want[1]) <= REL, (res, want)
    if not math.isnan(want[2]):
        assert rel_scalar(res[2], want[2]) <= REL
    got = lrn.core.get_named()
    for k in z:
        if k.startswith("p_out/"):
            refv = torch.from_numpy(z[k])
            if k == "p_out/log_alpha":
                assert (got["log_alpha"].reshape(-1) - refv.reshape(-1)).abs().max().item() <= 1e-6
            else:
                assert rel_l2(got[k[6:]].reshape(refv.shape), refv) <= REL, (k, rel_l2(got[k[6:]].reshape(refv.shape), refv))
    lrn.memory.stop()
