"""CPU: the n-step reference (oracle/nstep_ref.py) against brute force, and the trajectory stitcher."""
import pickle

import numpy as np
import pytest

import nstep_ref
import redis_stub
from _harness import _play, random_pushes
from distributed_sac_b200.stitch import Stitcher


@pytest.mark.parametrize("T,cap,streams,max_rows", [(0, 64, 5, 12), (0, 16, 3, 40), (3, 48, 6, 20), (4, 32, 9, 70)])
def test_ring_model_equals_list_of_trajectories(T, cap, streams, max_rows):
    """The incremental link rules give exactly the table the invariant defines, after every push: interleaved streams,
    terminals and cuts mid-stream, many wraps, pushes larger than a sub-ring, streams that change task, plain pushes."""
    rng = np.random.default_rng(cap + T)
    ring, brute = nstep_ref.RingModel(cap, T), nstep_ref.TrajectoryModel(cap, T)
    linked = 0
    for task, r, d, sid, cut in random_pushes(rng, 120, max(T, 1), streams, max_rows, plain_every=7):
        ring.push(task, r, d, sid, cut)
        brute.push(task, d, sid, cut)
        assert np.array_equal(ring.link, brute.links())
        linked += int((ring.link >= 0).sum())
    assert linked > 0
    # pred is the inverse of link wherever a link exists
    for t in range(ring.T):
        for i, j in enumerate(ring.link[t]):
            if j >= 0:
                assert ring.pred[t, j] == i


def test_fold_equals_fp64_nstep_return():
    rng = np.random.default_rng(0)
    for n in (1, 2, 3, 5, 16):
        for gamma in (0.99, 0.9, 0.5):
            L = 40
            r = rng.standard_normal(L).astype(np.float32)
            d = (rng.random(L) < 0.1).astype(np.float32)
            link = np.arange(1, L + 1, dtype=np.int32)
            link[-1] = -1
            link[d != 0] = -1                       # a terminal row has no successor
            R, disc, dd, last, m = nstep_ref.fold(r, d, link, L, np.arange(L), n, gamma)
            for i in range(L):
                end = i
                while d[end] == 0 and end + 1 < L:
                    end += 1
                want = nstep_ref.nstep_return_f64(r[i:end + 1], d[i:end + 1], gamma, n)
                assert abs(R[i] - want[0]) <= 1e-6 * max(1.0, abs(want[0]))
                assert abs(disc[i] - want[1]) <= 1e-6
                assert dd[i] == want[2] and m[i] == want[3] and last[i] == i + m[i] - 1
            if n == 1:
                assert np.array_equal(R, r) and np.all(disc == np.float32(gamma)) and np.array_equal(dd, d)


def test_stitcher_rebuilds_trajectories_from_interleaved_players():
    rng = np.random.default_rng(4)
    server = redis_stub.StrictRedis(host="nstep-stitch")
    server.delete("sample")
    rows = _play(rng, 3, 600, time_limit=25)
    st = Stitcher()
    got = []
    for k in range(0, len(rows), 37):               # drained in chunks, like the buffer thread
        for _who, payload in rows[k:k + 37]:
            server.rpush("sample", pickle.dumps(payload))
        pipe = server.pipeline()
        pipe.lrange("sample", 0, -1)
        pipe.ltrim("sample", -1, 0)
        datas, _ = pipe.execute()
        data = [pickle.loads(x) for x in datas]
        got.extend(st.assign(np.stack([x[0] for x in data]), np.stack([x[3] for x in data]), [x[4] for x in data]))
        assert st.take_abandoned() == []
    # consecutive rows of one episode share a stream id; the rows of an episode form one unbroken run of that id
    last_of = {}
    for (p, ep, t), sid, (_, payload) in zip([w for w, _ in rows], got, rows):
        if t > 0:
            assert last_of[(p, ep)] == sid, "a trajectory was split"
        last_of[(p, ep)] = sid
    # two different open episodes never share an id at the same time
    open_id = {}
    for (p, ep, t), sid, (_, payload) in zip([w for w, _ in rows], got, rows):
        holder = open_id.get(sid)
        assert holder is None or holder == (p, ep), "two live trajectories share a stream id"
        open_id[sid] = (p, ep)
        if payload[4]:
            del open_id[sid]
    assert max(got) < 64, "ids are recycled"


def test_stitcher_evicts_oldest_and_reports_abandoned_ids():
    st = Stitcher(max_open=4)
    s = np.arange(10 * 3, dtype=np.float32).reshape(10, 3)
    ids = st.assign(s, s + 1000, np.zeros(10))          # ten trajectories that never continue
    assert len(set(ids)) == 10 and st.open_tails == 4
    gone = st.take_abandoned()
    assert sorted(gone) == sorted(ids[:6].tolist())
    again = st.assign(s + 5000, s + 6000, np.zeros(10))
    assert set(again[:6]) <= set(gone) | set(range(10, 20))    # closed ids may serve again only after take_abandoned()
    cont = st.assign((s + 6000)[-1:], s[:1], [True])    # continues the newest tail, then closes it
    assert cont[0] == again[-1]
