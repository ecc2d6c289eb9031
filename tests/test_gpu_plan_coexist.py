"""GPU: handles whose plans launch one kernel with different dynamic shared memory coexist in one process.  The limit a
kernel launches under is one per process, so a handle built later must leave it high enough for the plans of the handles
built before it.  The first handle steps through paths it had not captured yet when the second was built (b200sac_step
after sampled steps, then an eager profile_step) and must compute bit for bit what it computes alone."""
import dataclasses

import numpy as np
import pytest
import torch

import sac_port as sp
from _golden import core_config
from _harness import ADAM_M, ADAM_V, MTSAC_T4, PARAMS, SMALL, _bits, _inputs, cuda  # noqa: F401

pytestmark = pytest.mark.gpu


def _pcgrad(T):
    spec = sp.SacSpec(**dict(MTSAC_T4, num_tasks=T))
    return spec, dataclasses.replace(core_config(spec, precision=0), pcgrad=True)


def _cases():
    """id -> ((spec, config) of the first handle, config of the second)."""
    t4, t4_cfg = _pcgrad(4)
    return {
        # the per-layer plan launches head_bwd with dynamic shared memory, the layer-chained plan does not launch it
        "per_layer_then_chained": ((SMALL, core_config(SMALL, precision=1)), core_config(sp.ll_spec(), precision=0)),
        # pcgrad_kernel's shared memory grows with the task count
        "pcgrad_t4_then_t2": ((t4, t4_cfg), _pcgrad(2)[1]),
    }


def _run(spec, cfg, second_cfg):
    """The first handle's state after two sampled steps, one b200sac_step and one eager profile_step; with second_cfg, a
    second handle is built after the sampled steps and kept open until the end."""
    from distributed_sac_b200.core import Replay, SacCore
    core = SacCore(cfg, 0, seed=3)
    ring = Replay(core, 8 * spec.batch, "device", seed=5)
    ring.fill_synthetic(8 * spec.batch, seed=7)
    core.step_sampled(ring, 2)
    torch.cuda.synchronize()
    second = SacCore(second_cfg, 0, seed=4) if second_cfg is not None else None
    b, e1, e2 = _inputs(spec, False, 1, 0)
    core.step(*[x.cuda() for x in b], e1.cuda(), e2.cuda())
    core.profile_step(ring, iters=1)
    torch.cuda.synchronize()
    out = [_bits(core.export_arena(which).numpy()) for which in (PARAMS, ADAM_M, ADAM_V)]
    out.append(_bits(core.read_losses(4).numpy()))
    ring.close()
    core.close()
    if second is not None:
        second.close()
    return out


@pytest.mark.parametrize("case", sorted(_cases()))
def test_earlier_handle_steps_after_a_later_one_is_built(cuda, case):
    (spec, cfg), second_cfg = _cases()[case]
    alone = _run(spec, cfg, None)
    beside = _run(spec, cfg, second_cfg)
    for what, a, b in zip(("parameters", "Adam m", "Adam v", "losses"), alone, beside):
        assert np.array_equal(a, b), f"{case}: {what} differ from the handle's steps alone"
