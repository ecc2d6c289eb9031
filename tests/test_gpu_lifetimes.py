"""GPU: every CUDA resource of a handle, a ring and a library call is released -- on success, on failure and on destroy.

Free device memory (torch.cuda.mem_get_info after a synchronize) must come back to where it was.  It is device-wide and
the GPU may be shared, so a reading over the tolerance is taken once more before it counts: a leak shows up again."""
import ctypes as C

import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import care_core_config, core_config
from _harness import cuda

pytestmark = pytest.mark.gpu

MiB = 1 << 20
TOL = 512 * MiB
ERR_NOMEM = -3          # B200SAC_ERR_NOMEM (include/b200sac.h)


def _free():
    torch.cuda.synchronize()
    return torch.cuda.mem_get_info()[0]


def _check_released(case):
    """case() does some work; the free memory it leaves must be within TOL of the free memory before it."""
    drops = []
    for _ in range(2):
        before = _free()
        case()
        drops.append(before - _free())
        if drops[-1] <= TOL:
            return
    pytest.fail(f"free device memory dropped by {drops[0] / MiB:.0f} MiB, then by {drops[1] / MiB:.0f} MiB on the repeat")


def test_graph_timeline_on_an_empty_ring_releases_its_stamp_buffers(cuda):
    """The timeline's stamp buffers (8 bytes per launch and step, ~300 MB at 2^22 steps of an LL handle) are allocated
    before the ring is found not ready; nothing is launched."""
    from distributed_sac_b200.core import CoreConfig, Replay, SacCore
    core = SacCore(CoreConfig(), 0, seed=0)
    ring = Replay(core, capacity=4096, where="device", seed=1)

    def case():
        for _ in range(8):
            with pytest.raises(RuntimeError, match="replay not ready"):
                core.graph_timeline(ring, iters=1 << 22)

    _check_released(case)
    ring.close()
    core.close()


def test_create_failure_at_the_work_slab_releases_the_arenas(cuda):
    """A shape whose arenas fit but whose work slab cannot (one hidden layer of 2^21 units at batch 2048: ~190 GB of
    activations) fails with B200SAC_ERR_NOMEM and leaves nothing behind; a normal handle can be created right after."""
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import CoreConfig, SacCore, layout
    cfg = CoreConfig(actor_hidden=[1 << 21], critic_hidden=[1 << 21], batch=2048)
    _, arena, trainable = layout(cfg)
    arenas = 4 * (arena + 3 * trainable + 3 * trainable)     # params, Adam m / v, gradients and their 3 split-K slices
    if arenas + 2 * TOL > _free():
        pytest.skip(f"the arenas ({arenas / MiB:.0f} MiB) do not fit in the free device memory")
    lib = _lib.load()

    def case():
        c, h = cfg.to_c(), C.c_void_p(0)
        rc = lib.b200sac_create(C.byref(c), 0, C.c_uint64(0), C.byref(h))
        assert rc == ERR_NOMEM and not h.value, (rc, lib.b200sac_last_error().decode())

    _check_released(case)
    core = SacCore(CoreConfig(), 0, seed=0)
    core.step_host(*sp.synthetic_batch(sp.SacSpec(), seed=1))
    core.close()


_CARE = cp.CareSpec(num_tasks=4, actor_hidden=[64, 64], critic_hidden=[64, 64], batch=40, num_encoders=3, mix_hidden=[24],
                    mix_out=12, ctx_hidden=[20], ctx_out=12, emb_dim=12)
HANDLES = {   # name -> (spec, core config): the layer-chained LL step, the per-layer 3xTF32 step, CARE(M), three replicas
    "chained_ll": (sp.SacSpec(), lambda s: core_config(s)),
    "per_layer_tf32": (sp.SacSpec(), lambda s: core_config(s, precision=1)),
    "care": (_CARE, lambda s: care_core_config(s, precision=1)),
    "replicas3": (sp.SacSpec(), lambda s: core_config(s, replicas=3)),
}
RINGS = {
    "device": dict(where="device"),
    "pinned host": dict(where="host"),
    "prioritized": dict(where="device", prioritized=dict(alpha=0.6, beta=0.4, eps=1e-6)),
    "linked": dict(where="device", trajectories=True),
}


def _use_and_destroy(name, seed):
    """Create one handle and one ring of every kind, run everything that allocates, destroy the rings, then the handle."""
    from distributed_sac_b200.core import Replay, SacCore
    spec, cfg = HANDLES[name]
    core = SacCore(cfg(spec), 0, seed=seed)
    R = core.cfg.replicas
    batch = (cp if name == "care" else sp).synthetic_batch(spec, seed=seed, batch=R * spec.batch)
    core.step(*[t.to(core.device) for t in batch])
    core.step_host(*batch)
    for image_bytes in (64, 4096):      # the second template replaces the first one's images and index maps
        core.blob_template(bytes(image_bytes), [], extra=("log_alpha",))
    core.blob_begin()
    blob, extra = core.blob_wait()
    assert len(blob) == 4096 and extra["log_alpha"].size == max(spec.num_tasks, 1)
    rings = {kind: Replay(core, capacity=4096, seed=seed, **kw) for kind, kw in RINGS.items()}
    for kind, ring in rings.items():
        ring.fill_synthetic(4096, seed=seed)
        core.prepare(ring)
        core.step_sampled(ring, 3)
        if kind != "pinned host":        # eager and in-graph timing runs need a device ring
            core.profile_step(ring, iters=2)
            core.graph_timeline(ring, iters=2)
    for ring in rings.values():
        ring.close()
    core.close()


@pytest.mark.parametrize("name", list(HANDLES))
def test_repeated_create_use_destroy_releases_everything(cuda, name):
    _use_and_destroy(name, seed=0)      # first use: module loading and the context's own growth happen here

    def case():
        for cycle in range(10):
            _use_and_destroy(name, seed=1 + cycle)

    _check_released(case)
