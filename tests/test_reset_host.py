"""Host side of network resets: the ctypes mirrors of b200sac_reset_part / b200sac_reset_spec, and SacCore.reset's
keyword-to-struct conversion (reset_spec) and the learner's argument checks, none of which needs a GPU."""
import json
import math
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
HDR = open(os.path.join(ROOT, "include", "b200sac.h")).read()


def _fields(struct):
    body = re.search(r"typedef struct %s \{(.*?)\} %s;" % (struct, struct), HDR, re.S).group(1)
    body = re.sub(r"/\*.*?\*/", "", body, flags=re.S)
    return [decl.split() for decl in body.split(";") if decl.strip()]


def test_reset_structs_match_header():
    from distributed_sac_b200 import _lib
    C = _lib.C
    ctype = {"int32_t": C.c_int32, "double": C.c_double}
    declared = [(name, ctype[t]) for t, name in _fields("b200sac_reset_part")]
    assert [(n, t) for n, t in _lib.ResetPart._fields_] == declared
    (t, name), = _fields("b200sac_reset_spec")
    assert (t, name) == ("b200sac_reset_part", "part[B200SAC_RESET_PARTS]")
    assert _lib.ResetSpec._fields_ == [("part", _lib.ResetPart * _lib.RESET_PARTS)]
    assert C.sizeof(_lib.ResetPart) == 16 and C.sizeof(_lib.ResetSpec) == 16 * 5


def test_reset_part_indices_match_header():
    from distributed_sac_b200 import _lib
    from distributed_sac_b200.core import RESET_PARTS
    enum = dict(re.findall(r"B200SAC_RESET_(\w+) = (\d+)", HDR))
    assert {k: int(v) for k, v in enum.items()} == {
        "ACTOR": _lib.RESET_ACTOR, "CRITIC": _lib.RESET_CRITIC, "ALPHA": _lib.RESET_ALPHA, "ENCODER": _lib.RESET_ENCODER,
        "CONTEXT": _lib.RESET_CONTEXT, "PARTS": _lib.RESET_PARTS}
    assert [RESET_PARTS.index(k.lower()) for k in ("ACTOR", "CRITIC", "ALPHA", "ENCODER", "CONTEXT")] == \
        [int(enum[k]) for k in ("ACTOR", "CRITIC", "ALPHA", "ENCODER", "CONTEXT")]


def _cfgs():
    from distributed_sac_b200.core import CoreConfig
    return dict(sac=CoreConfig(actor_hidden=[64, 48, 32], critic_hidden=[40]),
                care_m=CoreConfig(num_tasks=4, batch=64, care=True),
                care_o=CoreConfig(num_tasks=4, batch=64, care=True, care_original=True))


def _layers(spec):
    return [spec.part[i].layers for i in range(5)]


def _shrinks(spec):
    return [spec.part[i].shrink for i in range(5)]


def test_default_is_a_full_reset_of_the_parts_the_handle_has():
    from distributed_sac_b200.core import reset_spec
    c = _cfgs()
    assert _layers(reset_spec(c["sac"])) == [4, 2, 1, 0, 0]
    assert _layers(reset_spec(c["care_m"])) == [3, 3, 1, 1, 0]
    assert _layers(reset_spec(c["care_o"])) == [3, 3, 1, 1, 1]
    assert _shrinks(reset_spec(c["sac"])) == [0.0] * 5


def test_parts_and_shrink_fill_the_struct():
    from distributed_sac_b200.core import reset_spec
    c = _cfgs()
    s = reset_spec(c["sac"], actor=1, critic="all")
    assert _layers(s) == [1, 2, 0, 0, 0]
    s = reset_spec(c["care_o"], 0.25, critic=7, alpha=True, context=True, encoder=False)
    assert _layers(s) == [0, 7, 1, 0, 1] and _shrinks(s) == [0.25] * 5
    s = reset_spec(c["care_m"], {"critic": 0.5, "encoder": 1.0}, critic=2, encoder=True, actor=0)
    assert _layers(s) == [0, 2, 0, 1, 0] and _shrinks(s) == [0.0, 0.5, 0.0, 1.0, 0.0]
    assert _layers(reset_spec(c["sac"], encoder=False, context=0, alpha=1)) == [0, 0, 1, 0, 0]


@pytest.mark.parametrize("kw", [
    dict(actor=-1), dict(critic=True), dict(actor=1.5), dict(critic="most"), dict(alpha=2), dict(alpha="yes"),
    dict(encoder=True), dict(context=True), dict(reset_actor=1), dict(shrink=1.5), dict(shrink=-0.1),
    dict(shrink=math.nan), dict(shrink=True), dict(shrink="0.5"), dict(shrink={"bogus": 0.1}),
    dict(shrink={"actor": 2.0}), dict(shrink={"critic": math.nan}),
])
def test_bad_arguments_raise_value_error(kw):
    from distributed_sac_b200.core import reset_spec
    with pytest.raises(ValueError):
        reset_spec(_cfgs()["sac"], **kw)


def test_context_needs_care_o():
    from distributed_sac_b200.core import reset_spec
    with pytest.raises(ValueError):
        reset_spec(_cfgs()["care_m"], context=True)
    reset_spec(_cfgs()["care_m"], encoder=True)


@pytest.mark.parametrize("kw", [dict(reset_interval=0), dict(reset_interval=2.5), dict(reset_interval=True),
                                dict(reset=dict(actor=1)), dict(reset_interval=5, reset=dict(encoder=True)),
                                dict(reset_interval=5, reset=dict(actor=-2)), dict(reset_interval=5, reset=dict(net=1))])
def test_learner_refuses_bad_reset_arguments_before_building_a_handle(tmp_path, kw):
    import redis_stub
    from distributed_sac_b200 import learner as L
    p = tmp_path / "ll.json"
    p.write_text(json.dumps({"device": "cuda", "buffer_size": 1e5, "reward_scale": 1, "batch_size": 64, "gamma": 0.99,
                             "lr_actor": 3e-4, "lr_critic": 3e-4, "log_alpha": 0, "tau": 0.005, "start_memory_len": 1000}))
    with pytest.raises(ValueError):
        L.LunarLanderLearner(str(p), write_mode=False, server=redis_stub.StrictRedis(host=str(tmp_path)), **kw)
