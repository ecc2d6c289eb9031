"""GPU: n-step returns on the device ring -- trajectory links kept at push time, the return folded in the step's gather,
per-replica horizon (include/b200sac.h, csrc/nstep_kernels.cuh) against oracle/nstep_ref.py and the autograd oracle."""
import dataclasses
import json
import os
import pickle

import numpy as np
import pytest
import torch

import care_port as cp
import nstep_ref
import per_ref
import redis_stub
import sac_port as sp
from _golden import REL, check_forced, check_port_state, cuda_relu_masks, rel_scalar, sync_core_to_port
from _harness import (LL_CFG, MTSAC_T4, PER_LAYER, SMALL, VS400, _core, _play, _tasks, capture_grads, care_t4, check_adam,
                      check_grads, cuda, new_model, random_pushes, snapshot)

pytestmark = pytest.mark.gpu

PER = dict(alpha=0.6, beta=0.4, eps=1e-6)
INVALID, STATE = -1, -4


def _spec(name):
    """(spec, care, precision): LunarLander (layer-chained plan), the VSAC shape at both precisions (per-layer plan), a
    per-layer learner, MTSAC with weighted loss, small CARE(M)."""
    if name == "chained":
        return sp.ll_spec(), False, 0
    if name in ("vsac_p0", "vsac_p1"):
        return sp.SacSpec(**VS400), False, int(name[-1])
    if name in ("per_layer_p0", "per_layer_p1"):
        return sp.SacSpec(**PER_LAYER), False, int(name[-1])
    if name in ("mtsac", "mtsac_p0"):
        return sp.SacSpec(**MTSAC_T4), False, 0 if name.endswith("_p0") else 1
    if name == "tiny":
        return dataclasses.replace(SMALL, batch=8), False, 0
    if name == "tiny_mt":
        return dataclasses.replace(SMALL, batch=8, num_tasks=4), False, 0
    return care_t4(), True, 1


def _episodes(spec, care, n, seed, n_streams=7, p_done=0.05, p_cut=0.03):
    """n synthetic transitions in push order with interleaved streams: (s, a, r, s2, d) tensors, stream ids, cut flags."""
    s, a, r, s2, d = (cp if care else sp).synthetic_batch(spec, seed=seed, batch=n)
    rng = np.random.default_rng(seed)
    d = torch.from_numpy((rng.random(n) < p_done).astype(np.float32)).reshape(n, 1)
    sid = rng.integers(n_streams, size=n)
    if spec.num_tasks > 0:                      # a player works on one task: its rows stay in one sub-ring
        sid = sid * spec.num_tasks + _tasks(spec, s)
    return (s, a, r, s2, d), sid.astype(np.int32), (rng.random(n) < p_cut).astype(np.uint8)


class Mirror:
    """nstep_ref.RingModel of one replica's ring plus the host table [ring index] -> the five row tensors."""

    def __init__(self, spec, cap):
        self.spec, self.cap = spec, cap
        self.model = nstep_ref.RingModel(cap, spec.num_tasks)
        self.table = None

    def push(self, rows, stream=None, cut=None):
        s, a, r, s2, d = rows
        if self.table is None:
            self.table = [torch.zeros(self.cap, x.shape[1]) for x in rows]
        task = _tasks(self.spec, s)
        slot = self.model.push(task, r.reshape(-1).numpy(), d.reshape(-1).numpy(), stream, cut)
        keep = slot >= 0
        where = torch.from_numpy(task[keep] * self.model.cap_t + slot[keep])
        for t, x in zip(self.table, rows):
            t[where] = x[torch.from_numpy(keep)]

    def fold_batch(self, idx, n, gamma):
        """The folded minibatch of ring indices idx: (s, a, R, s2, d) tensors, disc, m."""
        R, disc, d, last, m = self.model.fold(idx, n, gamma)
        s, a, _r, s2, _d = self.table
        idx, last = torch.as_tensor(idx).long(), torch.from_numpy(last)
        return [s[idx], a[idx], torch.from_numpy(R).reshape(-1, 1), s2[last], torch.from_numpy(d).reshape(-1, 1)], disc, m


def _ring(core, spec, care, cap, n, seed=5, prioritized=None, trajectories=True, ring_seed=1, replicas=1, chunk=997):
    """A ring filled by pushes of `chunk` rows with stream ids (plain pushes on an unlinked ring), and its Mirror."""
    from distributed_sac_b200.core import Replay
    rb = Replay(core, cap, seed=ring_seed, prioritized=prioritized, trajectories=trajectories)
    rows, sid, cut = _episodes(spec, care, n, seed)
    mirror = Mirror(spec, cap)
    for k in range(0, n, chunk):
        part = [x[k:k + chunk] for x in rows]
        for rep in range(replicas):
            if trajectories:
                rb.push(*[x.numpy() for x in part], replica=rep, stream=sid[k:k + chunk], cut=cut[k:k + chunk])
            else:
                rb.push(*[x.numpy() for x in part], replica=rep)
        mirror.push(part, sid[k:k + chunk], cut[k:k + chunk])
    return rb, mirror


# ---- 1. nothing changes at n = 1 -----------------------------------------------------------------------------------
@pytest.mark.parametrize("prioritized", [None, PER], ids=["uniform", "per"])
@pytest.mark.parametrize("name", ["chained", "vsac_p0", "vsac_p1", "mtsac", "care_m"])
def test_linked_ring_at_n1_is_bit_identical(cuda, name, prioritized):
    """A linked ring with horizon 1 and an unlinked ring, same seed and pushes: losses and every parameter, target and
    Adam-moment tensor are identical bit for bit after 16 steps, and a step launches the same number of kernels."""
    spec, care, precision = _spec(name)
    a, b = _core(spec, care, precision), _core(spec, care, precision)
    ra, _ = _ring(a, spec, care, 4096, 4096, prioritized=prioritized, trajectories=False)
    rb, mirror = _ring(b, spec, care, 4096, 4096, prioritized=prioritized, trajectories=True)
    assert (mirror.model.link >= 0).sum() > 1000 and rb.get_nstep() == 1
    a.step_sampled(ra, 16)
    b.step_sampled(rb, 16)
    for which in (0, 1, 2):
        assert torch.equal(a.export_arena(which), b.export_arena(which)), (name, which)
    assert torch.equal(a.read_losses(16), b.read_losses(16))
    assert a.launches_per_step == b.launches_per_step
    assert a.get_steps() == b.get_steps()
    assert np.all(b.debug("nstep_m").numpy() == 1)
    assert torch.equal(b.debug("disc"), torch.full((spec.batch,), np.float32(spec.gamma)))
    for x in (ra, rb, a, b):
        x.close()


# ---- 2. links ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cap,streams,max_rows,prioritized", [("tiny", 64, 5, 12, None), ("tiny", 32, 3, 80, PER),
                                                                  ("tiny_mt", 48, 6, 20, None), ("tiny_mt", 32, 9, 70, None)])
def test_links_equal_reference_after_random_pushes(cuda, name, cap, streams, max_rows, prioritized):
    """b200sac_replay_get_links equals the ring model after every push of a random sequence: interleaved streams, d and
    cut mid-stream, several wraps, successors / predecessors / stream tails overwritten, pushes larger than the ring, task
    sub-rings (streams that change task), plain pushes mixed in."""
    from distributed_sac_b200.core import Replay
    spec, care, precision = _spec(name)
    core = _core(spec, care, precision)
    rb = Replay(core, cap, prioritized=prioritized, trajectories=True)
    model = nstep_ref.RingModel(cap, spec.num_tasks)
    T = max(spec.num_tasks, 1)
    rng = np.random.default_rng(cap)
    for task, r, d, sid, cut in random_pushes(rng, 60, T, streams, max_rows, plain_every=7):
        n = len(task)
        s = rng.standard_normal((n, spec.obs_dim)).astype(np.float32)
        if spec.num_tasks:
            s[:, spec.state_dim:] = np.eye(T, dtype=np.float32)[task]
        a = rng.standard_normal((n, spec.act_dim)).astype(np.float32)
        rb.push(s, a, r, s.copy(), d, stream=sid, cut=cut)
        model.push(task, r, d, sid, cut)
        for t in range(T):
            assert np.array_equal(rb.links(t), model.link[t]), (name, t)
    assert (model.link >= 0).sum() > 0
    rb.close()
    core.close()


# ---- 3. fold -----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,cap,n_rows", [("chained", 4096, 6000), ("mtsac", 4096, 3000)])
def test_fold_of_every_slot_equals_reference(cuda, name, cap, n_rows):
    """fold over every filled slot equals the reference bit for bit (R, disc, d, s', m) for n in {1, 2, 3, 5, 16}, on
    replicas with different horizons and different gamma (the ring wrapped for the LunarLander case)."""
    spec, care, precision = _spec(name)
    core = _core(spec, care, precision, replicas=2)
    rb, mirror = _ring(core, spec, care, cap, n_rows, replicas=2)
    idx = mirror.model.filled()
    for n0, n1, g0, g1 in ((1, 16, 0.99, 0.9), (2, 3, 0.95, 0.99), (5, 1, 0.5, 0.997)):
        rb.set_nstep(n0, replica=0)
        rb.set_nstep(n1, replica=1)
        core.set_hparams(0, gamma=g0)
        core.set_hparams(1, gamma=g1)
        assert (rb.get_nstep(0), rb.get_nstep(1)) == (n0, n1)
        hops = 0
        for rep, n, g in ((0, n0, g0), (1, n1, g1)):
            s, a, R, s2, d, disc, m = rb.fold(idx, replica=rep)
            want, wdisc, wm = mirror.fold_batch(idx, n, g)
            assert np.array_equal(R, want[2].reshape(-1).numpy()) and np.array_equal(disc, wdisc) and np.array_equal(m, wm)
            assert np.array_equal(d, want[4].reshape(-1).numpy())
            assert np.array_equal(s, want[0].numpy()) and np.array_equal(a, want[1].numpy()) and np.array_equal(s2, want[3].numpy())
            assert m.max() <= n
            hops = max(hops, int(m.max()))
        assert hops >= min(max(n0, n1), 3), "the chains are too short to exercise the fold"
    rb.close()
    core.close()


# ---- 4. the step trains on the fold ------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,prioritized", [("chained", None), ("chained", PER), ("per_layer_p0", None), ("per_layer_p1", None),
                                              ("mtsac", None), ("mtsac_p0", None)])
def test_step_matches_oracle_on_the_folded_minibatch(cuda, name, prioritized):
    """With n = 3 and 5 the step's "r", "d", "disc", "nstep_m" equal the fold of its own "idx", and the step matches the
    autograd oracle fed the folded minibatch and the per-row discount (CUDA masks forced, kinks proven) at 1e-4: losses, y,
    Q and every parameter, target and Adam moment; on a prioritized ring also the leaf values of the n-step TD error."""
    spec, care, precision = _spec(name)
    core = _core(spec, care, precision)
    rb, mirror = _ring(core, spec, care, 4096, 4096, prioritized=None if prioritized is None else dict(PER, beta=1.0))
    port = sp.PortLearner(spec, sp.init_params(spec, seed=3))
    ref_grads = capture_grads(port)
    model = new_model(core)
    B, A = spec.batch, spec.act_dim
    for step, n in enumerate((3, 5, 3)):
        rb.set_nstep(n)
        sync_core_to_port(core, port)
        model[0].seed(list(core.get_steps()) + [0])
        before = snapshot(core, 0)
        core.step_sampled(rb, 1)
        act = model[0].bump()
        idx = core.debug("idx").long().numpy()
        batch, disc, m = mirror.fold_batch(idx, n, spec.gamma)
        assert np.array_equal(core.debug("r").numpy(), batch[2].reshape(-1).numpy())
        assert np.array_equal(core.debug("d").numpy(), batch[4].reshape(-1).numpy())
        assert np.array_equal(core.debug("disc").numpy(), disc) and np.array_equal(core.debug("nstep_m").numpy(), m)
        assert m.max() == n and m.min() < n, "the minibatch does not mix full and shortened horizons"
        f = rb.fold(idx)
        assert np.array_equal(f[2], batch[2].reshape(-1).numpy()) and np.array_equal(f[3], batch[3].numpy())
        eps = core.debug("psave").reshape(2 * B, A, 8)[:, :, 5]
        e1, e2 = eps[:B].clone(), eps[B:].clone()
        forced = cuda_relu_masks(core, spec)
        port.spec = dataclasses.replace(spec, gamma=torch.from_numpy(disc.copy()).reshape(B, 1))    # per-row discount
        w = core.debug("isw") if prioritized else torch.ones(B)
        with per_ref.ImportanceWeights(w), sp.ReluTape(forced) as tape:
            out = port.update_SAC(*batch, e1, e2, want_intermediates=True)
        port.spec = spec
        check_forced(tape, forced, f"{name} step {step}: ")
        L = core.read_losses(1)[0, 0]
        for j, want in enumerate((per_ref.weighted_critic_loss(out, w, spec.weighted_loss), out["actor_loss"])):
            assert rel_scalar(float(L[j]), want) <= REL, (name, step, j, float(L[j]), want)
        for key in ("y", "q1", "q2", "logp_next"):
            got, ref = core.debug(key), out[key].reshape(-1)
            assert float((got - ref).abs().max()) <= REL * (float(ref.abs().max()) + 1.0), (name, step, key)
        # the gradients the step consumed against the oracle's, and the optimizer step bit for bit
        check_grads(core, ref_grads, f"{name} step {step}")
        check_adam(core, model, 0, before, snapshot(core, 0, True), act, f"{name} step {step}")
        # The parameters themselves are compared only where Adam's g / (|g| + eps) map is well conditioned.  On 3xTF32 the
        # MTSAC run starts from zero biases, so after its first step a bias IS the update, and q2.1.bias[100] has
        # |g| = 1.29e-9 ~ eps/8: a gradient 1.7e-11 from the oracle's (that tensor passes the gradient check) moves its update
        # from 3.48e-5 to 3.44e-5 and the tensor to 1.3e-4 from the oracle.  The two checks above cover it exactly.
        check_port_state(core, port, params=name != "mtsac")
        if prioritized:
            y, q1, q2 = (out[k].reshape(-1).double() for k in ("y", "q1", "q2"))
            want_p = (((y - q1).abs() + (y - q2).abs()) / 2 + PER["eps"]) ** PER["alpha"]
            got_p = core.debug("prio").double()
            assert float(((got_p - want_p).abs() / want_p).max()) <= 1e-3
    rb.close()
    core.close()


# ---- 5. stream order -------------------------------------------------------------------------------------------------
def test_set_nstep_between_graph_launches(cuda):
    """24 steps enqueued as multi-step graphs with set_nstep and set_hparams(gamma=) between them equal, bit for bit, the
    same schedule run one step per call on a fresh handle."""
    spec, care, precision = _spec("chained")
    cores = [_core(spec, care, precision, replicas=2) for _ in range(2)]
    rings = [_ring(c, spec, care, 4096, 4096, replicas=2)[0] for c in cores]
    cores[0].prepare(rings[0])
    for k, (n0, n1, g) in enumerate(((1, 3, 0.99), (5, 2, 0.9), (16, 1, 0.97))):
        for c, r in zip(cores, rings):
            r.set_nstep(n0, replica=0)
            r.set_nstep(n1, replica=1)
            c.set_hparams(k % 2, gamma=g)
        cores[0].step_sampled(rings[0], 8)
        for _ in range(8):
            cores[1].step_sampled(rings[1], 1)
    for which in (0, 1, 2):
        for rep in range(2):
            assert torch.equal(cores[0].export_arena(which, rep), cores[1].export_arena(which, rep)), (which, rep)
    assert torch.equal(cores[0].read_losses(24), cores[1].read_losses(24))
    assert int(cores[0].debug("nstep_m", 0).max()) > 3 and int(cores[0].debug("nstep_m", 1).max()) == 1
    for x in rings + cores:
        x.close()


# ---- 6. refusals ---------------------------------------------------------------------------------------------------
def test_refusals_leave_everything_unchanged(cuda):
    import ctypes as C
    from distributed_sac_b200.core import Replay
    spec, care, precision = _spec("tiny")
    core = _core(spec, care, precision)
    lib = core.lib
    host = Replay(core, 64, where="host")
    assert lib.b200sac_replay_enable_trajectories(host._h) == INVALID
    with pytest.raises(ValueError):
        Replay(core, 64, where="host", trajectories=True)
    plain = Replay(core, 64)
    n32 = C.c_int32(7)
    assert lib.b200sac_replay_set_nstep(plain._h, 0, 3, None) == STATE
    assert lib.b200sac_replay_get_nstep(plain._h, 0, C.byref(n32)) == STATE and n32.value == 7
    rows, sid, cut = _episodes(spec, care, 40, 1)
    arrs = [np.ascontiguousarray(x.numpy()) for x in rows]
    ptrs = [C.c_void_p(x.ctypes.data) for x in arrs]
    assert lib.b200sac_replay_push_traj(plain._h, 0, 40, *ptrs, C.c_void_p(sid.ctypes.data), None) == STATE
    assert plain.size() == 0
    plain.push(*arrs)
    assert lib.b200sac_replay_enable_trajectories(plain._h) == STATE            # not empty
    rb = Replay(core, 64, trajectories=True)
    assert lib.b200sac_replay_enable_trajectories(rb._h) == STATE               # already linked
    rb.push(*arrs, stream=sid, cut=cut)
    links, size = rb.links().copy(), rb.size()
    for bad in (0, 17, -1):
        assert lib.b200sac_replay_set_nstep(rb._h, 0, bad, None) == INVALID
    assert lib.b200sac_replay_set_nstep(rb._h, 1, 2, None) == INVALID           # replica out of range
    assert rb.get_nstep() == 1
    for bad in (65536, -1):
        sid2 = sid.copy()
        sid2[17] = bad
        assert lib.b200sac_replay_push_traj(rb._h, 0, 40, *ptrs, C.c_void_p(sid2.ctypes.data), None) == INVALID
    assert lib.b200sac_replay_push_traj(rb._h, 0, 40, *ptrs, None, None) == INVALID
    out = np.empty(63, np.int32)
    assert lib.b200sac_replay_get_links(rb._h, 0, 0, 63, C.c_void_p(out.ctypes.data)) == INVALID
    assert lib.b200sac_replay_get_links(rb._h, 0, 1, 64, C.c_void_p(out.ctypes.data)) == INVALID
    with pytest.raises(RuntimeError):
        rb.fold([40])                                                           # an empty slot
    with pytest.raises(RuntimeError):
        rb.fold([64])
    assert np.array_equal(rb.links(), links) and rb.size() == size
    torch.cuda.synchronize()
    for x in (host, plain, rb, core):
        x.close()


# ---- 7. learner ------------------------------------------------------------------------------------------------------

def test_learner_stitches_interleaved_players(cuda, tmp_path):
    """LunarLanderLearner(replay_where="device", n_step=3) fed through the Redis stub by interleaved players runs update(),
    and its ring's links are the players' true trajectories."""
    from distributed_sac_b200.learner import LunarLanderLearner
    p = tmp_path / "cfg.json"
    p.write_text(json.dumps(LL_CFG))
    os.chdir(tmp_path)
    with pytest.raises(ValueError):
        LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path) + "x"), n_step=3)
    server = redis_stub.StrictRedis(host=str(tmp_path))
    lrn = LunarLanderLearner(str(p), write_mode=False, server=server, replay_where="device", buffer_size=4096, n_step=3)
    lrn.memory.stop()
    lrn.memory.join()
    rows = _play(np.random.default_rng(11), 4, 2000, time_limit=40)
    for k in range(0, len(rows), 173):
        for _who, payload in rows[k:k + 173]:
            server.rpush("sample", pickle.dumps(payload))
        lrn.memory.drain_once()
    want = np.full(4096, -1, np.int32)
    at = {who: i for i, (who, _) in enumerate(rows)}
    for i, ((pl, ep, t), payload) in enumerate(rows):
        if not payload[4] and (pl, ep, t + 1) in at:
            want[i] = at[(pl, ep, t + 1)]
    assert np.array_equal(lrn.memory.ring.links(), want) and (want >= 0).sum() > 1500
    assert lrn.memory.ring.get_nstep() == 3
    losses = lrn.update()
    assert all(np.isfinite(float(x)) for x in losses[:2])
    m = lrn.core.debug("nstep_m").numpy()
    assert m.max() == 3 and m.min() >= 1
    lrn.set_n_step(5)
    lrn.update()
    assert lrn.core.debug("nstep_m").numpy().max() == 5
    lrn.memory.ring.close()
    lrn.core.close()
