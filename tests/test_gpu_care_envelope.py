"""The CARE step (care_kernels.cuh; care_encode / the mixture backward / care_encode_rows in b200sac.cu) over the configurations
check_cfg accepts, against the autograd oracle (oracle/care_port.py).

The reference's CARE shapes (state 39, ctx_in 768, one mixture hidden layer of 50, K = 6, T = 10) reach few of the kernels'
branches.  The cases below walk the edges where they do branch:
  care_mixfwd_kernel      1, 2, 3 mixture hidden layers (ha / hb ping-pong, ha reused at layer 2); layers wider than 64 (two
                          o0 passes, the second partial); K > 6 (more than one (encoder, 8-row) task per warp); partial 32-row CTAs
  step-plan fallback      more than 4 mixture layers, or weights beyond 225 KB: grouped mixture GEMMs (wgmma at precision 1)
                          and care_mix_kernel; split-K on 2K mixture gradient problems
  care_tables_kernel      narrow inputs (<= 64) with more than 64 outputs (remainder loop); inputs taking only the tail loop,
                          only the 8-wide loop, or the 24-, 8-wide and tail loops with lanes splitting; ctx_in 2048 (xe full);
                          CARE(O) trunks reading a 256-wide context code
  care_tab_reduce_kernel  K + ctx_out > 64 (several 64-value passes)
  care_mix(_bwd), softmax K = 1 (attention identically 1, trunk gradient exactly 0) and K = 32
  care_tab_wgrad_kernel   9-layer trunk / context nets; up to 64 tasks whose backward chains exceed 48 KiB (taken in chunks)
Every step is checked with the CUDA step's ReLU masks forced into the oracle (tests/_golden.py::kink_checked_step): losses,
every parameter / target / Adam moment, and every per-row output element by element.  Guards keep the sweep from passing
vacuously: the plan each case is meant to take is read back from the handle, every hidden layer is partly active, every
trainable tensor moves.  test_sweep_covers_every_branch mirrors the kernels' branch rules and names any branch the cases
stop reaching.
"""
import re

import pytest
import torch

import care_port as cp
import sac_port as sp
from _golden import check_forced, check_port_state, cuda_relu_masks, sync_core_to_port
from _harness import (CARE_ROW_OUTPUTS, _bad_elements, _core, _eps, _pad4, _params, _raise_bad, check_active, check_losses,
                      check_rows, cuda, plan_labels, run_checked)

gpu = pytest.mark.gpu

# reference encoder widths (MT10_Distributed_CARE_cfg.json encoder block)
_REF = dict(num_encoders=6, mix_hidden=[50], mix_out=50, ctx_in=768, ctx_hidden=[50, 50], ctx_out=50)
_MLP = dict(actor_hidden=[64, 48], critic_hidden=[56, 64])
_O = dict(modified=False, weighted_loss=False)

# id -> CareSpec fields.  cmf = care_mixfwd_kernel's shared memory, tab = care_tab_wgrad_kernel's chains of all tasks.
#   k1_t1         one encoder and one task: softmax of one logit (trunk untouched on both sides); a 33 -> 70 table layer
#                 (remainder loop) and a 70-wide input (tail loop only); mix_out 9; a partial CTA in both mixfwd jobs
#   k32           K = 32 everywhere: 128 (encoder, 8-row) tasks over 24 warps; K + ctx_out = 72; cmf 96 KB
#   nl3           two mixture hidden layers (ha -> hb); a 256-wide table input (one 8-wide pass); cmf 187 KB; action
#                 scale 2
#   deep4         three mixture hidden layers (ha reused); 68 / 72 / 66-wide layers (two o0 passes, the second partial);
#                 trunk 36 -> 72 (remainder loop); ctx_in 1000 (24-, 8-wide and tail loops, lanes split)
#   deep9         9 mixture layers: the fallback by depth; 9-layer trunk and context nets
#   smem_fb       weights of 300 KB: the fallback by size; obs 40, so mixture GEMMs take wgmma at precision 1; batch 512:
#                 split-K over 32 + 32 mixture gradient problems
#   tasks64_m     reference widths at 64 tasks: tab 51.5 KiB
#   mt50_o        CARE(O) at the reference widths with MT50's 50 tasks: tab 69.5 KiB
#   o_wide        CARE(O), emb = ctx_out = 256: a 512-wide header, a 256-wide trunk input, K + ctx_out = 261
#   o_deep        CARE(O), ctx_in 2048 (xe full), 6 context hidden layers: a 9-layer context encoder
#   tasks64_wide  64 tasks and widths near 512: tab 509 KB, eleven chunks of six tasks (the last one of four)
CASES = {
    "k1_t1": dict(state_dim=7, num_tasks=1, num_encoders=1, mix_hidden=[20], mix_out=9, ctx_in=33, ctx_hidden=[70], ctx_out=5,
                  batch=29),
    "k32": dict(state_dim=12, num_tasks=8, num_encoders=32, mix_hidden=[8], mix_out=8, ctx_in=768, ctx_hidden=[48], ctx_out=40,
                batch=200),
    "nl3": dict(state_dim=39, num_tasks=3, num_encoders=7, mix_hidden=[40, 24], mix_out=20, ctx_in=256, ctx_hidden=[100],
                ctx_out=20, batch=123, action_scale=2.0),
    "deep4": dict(state_dim=23, num_tasks=5, num_encoders=2, mix_hidden=[68, 36, 72], mix_out=66, ctx_in=1000,
                  ctx_hidden=[64, 65], ctx_out=30, batch=155),
    "deep9": dict(state_dim=39, num_tasks=3, num_encoders=4, mix_hidden=[16, 6, 32, 12, 8, 24, 40, 20], mix_out=14, ctx_in=64,
                  ctx_hidden=[24, 8, 40, 16, 12, 32, 20, 28], ctx_out=18, batch=99),
    "smem_fb": dict(state_dim=38, num_tasks=2, num_encoders=32, mix_hidden=[64], mix_out=48, ctx_in=200, ctx_hidden=[50],
                    ctx_out=40, batch=512),
    "tasks64_m": dict(state_dim=39, num_tasks=64, batch=128, **_REF),
    "mt50_o": dict(state_dim=39, num_tasks=50, batch=150, emb_dim=50, **_REF, **_O),
    "o_wide": dict(state_dim=17, num_tasks=7, num_encoders=5, mix_hidden=[40], mix_out=28, ctx_in=768, ctx_hidden=[],
                   ctx_out=256, emb_dim=256, batch=91, **_O),
    "o_deep": dict(state_dim=21, num_tasks=4, num_encoders=3, mix_hidden=[36], mix_out=20, ctx_in=2048,
                   ctx_hidden=[20, 8, 36, 16, 24, 10], ctx_out=12, emb_dim=12, batch=100, **_O),
    "tasks64_wide": dict(state_dim=10, num_tasks=64, num_encoders=8, mix_hidden=[500], mix_out=12, ctx_in=512,
                         ctx_hidden=[504, 496], ctx_out=480, batch=128),
}

def care_spec(name):
    return cp.CareSpec(**{**_MLP, **CASES[name]})


# ---------------------------------------------------------------------------------------------------------------------
# mirrors of the kernels' branch rules (care_kernels.cuh, care_encode in b200sac.cu)
# ---------------------------------------------------------------------------------------------------------------------
CMF_ROWS, CMF_RP, CMF_MAXL, CMF_WARPS = 32, 36, 4, 24
CMF_SMEM_MAX = 225 * 1024
TAB_WGRAD_FLOATS = 12288          # care_tab_wgrad_kernel's shared memory (kCareTabWgradSmemFloats)


def mixfwd_smem_floats(spec):
    """care_mixfwd_smem_floats: weights + biases, xs, ha (/ hb), zs, att."""
    K, dims = spec.num_encoders, cp.mix_dims(spec)
    n = sum(_pad4(K * o * i) + _pad4(K * o) for i, o in dims)
    n += dims[0][0] * CMF_RP
    n += (2 if len(dims) > 2 else 1) * K * max(o for _, o in dims) * CMF_RP
    n += K * CMF_ROWS * spec.mix_out + CMF_ROWS * (K + 1)
    return n + 8


def fused(spec):
    """care_encode takes care_mixfwd_kernel: at most 4 mixture layers whose shared-memory image fits 225 KB."""
    return len(cp.mix_dims(spec)) <= CMF_MAXL and 4 * mixfwd_smem_floats(spec) <= CMF_SMEM_MAX


def table_nets(spec):
    """(trunk, context net) layer dims as care_tables_kernel / care_tab_wgrad_kernel walk them."""
    return cp.trunk_dims(spec), (cp.ctx_dims(spec) if spec.modified else cp.cenc_dims(spec))


def table_branch(nin, nout):
    """Which of care_tables_kernel's dot-product loops a layer nin -> nout runs."""
    if nin <= 64:
        return "narrow+remainder" if nout > 64 else "narrow"
    lanes = set()
    for lane in range(32):
        i, used = lane, []
        if i + 23 * 32 < nin:
            used.append(24)
        while i + 23 * 32 < nin:
            i += 24 * 32
        if i + 7 * 32 < nin:
            used.append(8)
        while i + 7 * 32 < nin:
            i += 8 * 32
        if i < nin:
            used.append(1)
        lanes.add(tuple(used))
    loops = set().union(*lanes)
    if loops == {24, 8, 1} and len(lanes) > 1:
        return "24+8+tail, lanes split"
    if loops == {1}:
        return "tail only"
    if loops == {8}:
        return "8-wide only"
    return "24-wide" if 24 in loops else "8-wide + tail"


def tab_wgrad_floats_per_task(spec):
    trunk, ctx = table_nets(spec)
    return sum(o for _, o in trunk) + sum(o for _, o in ctx)


def tab_wgrad_chunks(spec):
    per = tab_wgrad_floats_per_task(spec)
    tc = max(1, min(spec.num_tasks, TAB_WGRAD_FLOATS // per))
    return -(-spec.num_tasks // tc)


def check_path(name, spec, precision):
    core = _core(spec, True, precision)
    labels = plan_labels(core)
    core.close()
    if fused(spec):
        assert "care_mixture_fwd+mix" in labels, f"{name}: expected the fused mixture kernel, plan {labels}"
        assert "care_mix" not in labels, f"{name}: fused case with a care_mix launch, plan {labels}"
    else:
        assert "care_mix" in labels and "care_mixture_fwd+mix" not in labels, f"{name}: expected the fallback, plan {labels}"
        first = labels[labels.index("care_tables") + 1:labels.index("care_mix")]
        assert len(first) >= len(cp.mix_dims(spec)) and all(n.startswith("gemm_fwd") for n in first), (name, first)
        if name == "smem_fb" and precision == 1:
            assert any("wgmma" in n for n in first), f"{name}: no wgmma GEMM among the mixture launches {first}"
    assert labels.count("care_tab_wgrad") == 1, labels
    return labels


# ---------------------------------------------------------------------------------------------------------------------
# 1: the oracle sweep, with the guards that it ran the intended plan on non-degenerate networks
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
@pytest.mark.parametrize("name", list(CASES))
def test_care_step_matches_oracle(cuda, name, precision):
    from distributed_sac_b200 import _lib
    spec = care_spec(name)
    check_path(name, spec, precision)
    p = _params(spec, 7, care=True)
    port = cp.CarePortLearner(spec, p)
    core = _core(spec, True, precision)
    what = f"{name} precision {precision}"
    flips, worst = run_checked(core, spec, port, 2, seed=13, what=what, care=True)
    got = core.get_named(_lib.PARAMS)
    gm, gv = core.get_named(_lib.ADAM_M), core.get_named(_lib.ADAM_V)
    ref, st = port.params(), port.adam_state()
    for k in port.trainable_names():
        if k.startswith("ase."):
            continue
        assert torch.isfinite(got[k]).all(), (what, k)
        if spec.num_encoders == 1 and k.startswith("cse.trunk."):
            # one attention logit: softmax is identically 1 and its gradient exactly 0 -- nothing may move, on either side
            assert torch.equal(got[k], p[k]) and torch.equal(ref[k], p[k]), f"{what}: {k} moved"
            for arena, mom in ((gm, st["m"]), (gv, st["v"])):
                assert not arena[k].any() and not mom[k].any(), f"{what}: Adam moment of {k} is not zero"
        else:
            assert not torch.equal(got[k], p[k]), f"{what}: {k} did not change in two steps"
    core.close()
    print(f"[kinks] {what}: {flips} mask bits differed, all at numerically-zero pre-activations")
    print(f"[rows] {what}: largest per-row |got - ref| / (|ref| + mean|ref|) = {worst:.2e}  "
          f"(fused {fused(spec)}, tab_wgrad chunks {tab_wgrad_chunks(spec)})")


# ---------------------------------------------------------------------------------------------------------------------
# 2: the sweep reaches every branch (the kernels' rules mirrored; no GPU needed)
# ---------------------------------------------------------------------------------------------------------------------
def test_sweep_covers_every_branch():
    have = set()
    for name in CASES:
        s = care_spec(name)
        nl = len(cp.mix_dims(s))
        if fused(s):
            have.add(f"fused nl={nl}")
            if s.num_encoders * (CMF_ROWS // 8) > CMF_WARPS:
                have.add("fused: more (encoder, 8-row) tasks than warps")
            if (2 * s.batch) % CMF_ROWS:
                have.add("fused: partial CTA in the 2B job")
            if s.batch % CMF_ROWS:
                have.add("fused: partial CTA in the B job")
            if any(o > 64 for _, o in cp.mix_dims(s)):
                have.add("fused: layer wider than 64")
        else:
            have.add("fallback by depth" if nl > CMF_MAXL else "fallback by size")
            if (s.state_dim + s.num_tasks) % 4 == 0 and s.batch >= 512:
                have.add("fallback: wgmma-eligible input rows, split-K mixture gradients")
        if s.num_encoders + s.ctx_out > 64:
            have.add("tab_reduce: several passes")
        if s.num_encoders in (1, 32):
            have.add(f"K={s.num_encoders}")
        for nin, nout in [d for net in table_nets(s) for d in net]:
            have.add(f"tables: {table_branch(nin, nout)}")
        if s.ctx_in == 2048:
            have.add("tables: ctx_in 2048")
        if not s.modified and s.emb_dim == 256:
            have.add("tables: 256-wide CARE(O) trunk input")
        if any(len(net) == 9 for net in table_nets(s)):
            have.add("tab_wgrad: 9-layer net")
        if 4 * s.num_tasks * tab_wgrad_floats_per_task(s) > 48 * 1024:
            have.add("tab_wgrad: chains above 48 KiB")
        if tab_wgrad_chunks(s) > 2:
            have.add("tab_wgrad: more than two chunks")
        have.add("CARE(M)" if s.modified else "CARE(O)")
    want = {"fused nl=2", "fused nl=3", "fused nl=4", "fallback by depth", "fallback by size",
            "fused: more (encoder, 8-row) tasks than warps", "fused: partial CTA in the 2B job", "fused: partial CTA in the B job",
            "fused: layer wider than 64", "fallback: wgmma-eligible input rows, split-K mixture gradients",
            "tab_reduce: several passes", "K=1", "K=32", "tables: narrow", "tables: narrow+remainder", "tables: tail only",
            "tables: 8-wide only", "tables: 24-wide", "tables: 24+8+tail, lanes split", "tables: ctx_in 2048",
            "tables: 256-wide CARE(O) trunk input", "tab_wgrad: 9-layer net", "tab_wgrad: chains above 48 KiB",
            "tab_wgrad: more than two chunks", "CARE(M)", "CARE(O)"}
    missing = sorted(want - have)
    assert not missing, f"no case reaches: {missing}"


def test_branch_mirrors():
    """The mirrors agree with the shapes worked out by hand in the case table."""
    assert 4 * mixfwd_smem_floats(care_spec("k32")) // 1024 == 95
    assert 4 * mixfwd_smem_floats(care_spec("nl3")) // 1024 == 187
    assert not fused(care_spec("smem_fb")) and not fused(care_spec("deep9")) and fused(care_spec("deep4"))
    assert table_branch(768, 50) == "24-wide" and table_branch(256, 100) == "8-wide only"
    assert table_branch(70, 5) == "tail only" and table_branch(1000, 64) == "24+8+tail, lanes split"
    assert table_branch(36, 72) == "narrow+remainder" and table_branch(64, 64) == "narrow"
    assert 4 * care_spec("tasks64_m").num_tasks * tab_wgrad_floats_per_task(care_spec("tasks64_m")) == 13184 * 4
    assert care_spec("mt50_o").num_tasks * tab_wgrad_floats_per_task(care_spec("mt50_o")) == 17800
    assert tab_wgrad_chunks(care_spec("tasks64_wide")) == 11 and tab_wgrad_chunks(care_spec("mt50_o")) == 2


# ---------------------------------------------------------------------------------------------------------------------
# 3: co-scheduled replicas with parameters and task ids of their own
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("precision", [0, 1], ids=["fp32", "tc3xtf32"])
def test_replicas_with_different_parameters_match_their_oracles(cuda, precision):
    """Three CARE(M) replicas, each its own parameter draw (embedding included) and minibatch: every replica follows its own
    oracle; at precision 0 each also equals bit for bit an R = 1 handle given the same state and inputs (at precision 1 the
    tensor-core split / tile choice depends on R)."""
    from distributed_sac_b200 import _lib
    spec = cp.CareSpec(state_dim=20, num_tasks=5, num_encoders=4, mix_hidden=[40], mix_out=24, ctx_in=100, ctx_hidden=[30],
                       ctx_out=16, batch=105, **_MLP)
    assert fused(spec) and spec.batch % CMF_ROWS
    R = 3
    params = [_params(spec, 30 + r, care=True) for r in range(R)]
    ports = [cp.CarePortLearner(spec, p) for p in params]
    batches = [cp.synthetic_batch(spec, seed=300 + r) for r in range(R)]
    gen = torch.Generator().manual_seed(3)
    eps = [_eps(spec, gen) for _ in range(R)]
    tids = [torch.argmax(b[0][:, -spec.num_tasks:], dim=1) for b in batches]
    assert not torch.equal(tids[0], tids[1]) and not torch.equal(tids[1], tids[2])

    core = _core(spec, True, precision, R)
    for r in range(R):
        sync_core_to_port(core, ports[r], r)
    core.step(*[torch.stack([b[j] for b in batches]) for j in range(5)],
              torch.stack([e[0] for e in eps]), torch.stack([e[1] for e in eps]))
    for r in range(R):
        forced = cuda_relu_masks(core, spec, r, care=True)
        with sp.ReluTape(forced) as tape:
            o = ports[r].update(*batches[r], *eps[r], want_intermediates=True)
        check_forced(tape, forced, f"replica {r}: ")
        check_active(core, spec, r, f"replica {r}: ", care=True)
        check_losses(core, o, r, f"replica {r}: ")
        check_port_state(core, ports[r], replica=r)
        check_rows(core, spec, o, r, f"replica {r}: ", CARE_ROW_OUTPUTS)
    L3 = core.read_losses(1)[0]
    assert not torch.equal(L3[0], L3[1]) and not torch.equal(L3[1], L3[2])

    if precision == 0:
        single = _core(spec, True, 0)
        for r in range(R):
            sync_core_to_port(single, cp.CarePortLearner(spec, params[r]))
            single.step(*batches[r], *eps[r])
            diff = [f"{which}:{k}" for which, arena in (("params", _lib.PARAMS), ("grads", _lib.GRADS), ("adam_m", _lib.ADAM_M),
                                                         ("adam_v", _lib.ADAM_V))
                    for a, b in [(core.get_named(arena, r), single.get_named(arena))] for k in a if not torch.equal(a[k], b[k])]
            assert not diff, f"replica {r} of the R = 3 handle differs from the R = 1 handle in {diff[:8]}"
            assert torch.equal(L3[r], single.read_losses(1)[0, 0]), (r, L3[r].tolist(), single.read_losses(1)[0, 0].tolist())
        single.close()
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 4: acting (b200sac_act): per-task tables, grouped SIMT mixture GEMMs and care_mix_kernel on n rows
# ---------------------------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", list(CASES))
def test_act_matches_oracle_policy(cuda, name):
    spec = care_spec(name)
    port = cp.CarePortLearner(spec, _params(spec, 11, care=True))
    core = _core(spec, True, 0)
    sync_core_to_port(core, port)
    B, A = spec.batch, spec.act_dim
    b0, b1 = cp.synthetic_batch(spec, seed=41), cp.synthetic_batch(spec, seed=42)
    obs = torch.cat([b0[0][: B // 2], b1[3][: B - B // 2]])                  # B rows of mixed tasks
    eps = torch.randn(B, A, generator=torch.Generator().manual_seed(4))
    with torch.no_grad():
        z = cp.context_encode(spec, port.p, torch.argmax(obs[:, -spec.num_tasks:], dim=1))
    for n in sorted({B, 1, (B // 3) | 1}):
        for stochastic in (True, False):
            e = eps[:n] if stochastic else torch.zeros(n, A)
            with torch.no_grad():
                ref = port._policy("ase", z[:n], obs[:n], e, False)[0].double()
            got = core.act(obs[:n], eps=e) if stochastic else core.act(obs[:n].cuda(), stochastic=False)
            bad, _ = _bad_elements(got, ref)
            if bad.any():
                _raise_bad(f"{name} act n={n} stochastic={stochastic}", bad, got.double(), ref)
    core.close()


# ---------------------------------------------------------------------------------------------------------------------
# 5: every bound of the accepted configurations: just inside is accepted, just outside is refused (host-side check)
# ---------------------------------------------------------------------------------------------------------------------
_EDGE_M = dict(care=True, state_dim=8, num_tasks=4, batch=64, num_encoders=4, mix_hidden=[16], mix_out=8, ctx_in=64,
               ctx_hidden=[16], ctx_out=8)
_EDGE_O = dict(_EDGE_M, care_original=True, ctx_out=16, emb_dim=16)
BOUNDS = {   # id -> (accepted, refused, message fragment)
    "num_encoders": (dict(_EDGE_M, num_encoders=32), dict(_EDGE_M, num_encoders=33), "num_encoders"),
    "num_tasks": (dict(_EDGE_M, num_tasks=64, batch=128), dict(_EDGE_M, num_tasks=65, batch=130), "num_tasks"),
    "mix_width": (dict(_EDGE_M, mix_hidden=[512]), dict(_EDGE_M, mix_hidden=[513]), "mix_hidden"),
    "mix_out": (dict(_EDGE_M, mix_out=512), dict(_EDGE_M, mix_out=513), "widths"),
    "ctx_width": (dict(_EDGE_M, ctx_hidden=[512]), dict(_EDGE_M, ctx_hidden=[513]), "ctx_hidden"),
    "ctx_in": (dict(_EDGE_M, ctx_in=2048), dict(_EDGE_M, ctx_in=2049), "ctx_in"),
    "o_ctx_layers": (dict(_EDGE_O, ctx_hidden=[16] * 6), dict(_EDGE_O, ctx_hidden=[16] * 7), "context-encoder layers"),
    "o_emb_dim": (dict(_EDGE_O, emb_dim=16), dict(_EDGE_O, emb_dim=15), "must equal"),
    "k_plus_ctx_out": (dict(_EDGE_M, num_encoders=32, ctx_out=480), dict(_EDGE_M, num_encoders=32, ctx_out=481),
                       "num_encoders + ctx_out"),
}


@pytest.mark.parametrize("bound", list(BOUNDS))
def test_bounds_of_the_accepted_configurations(bound):
    from distributed_sac_b200.core import CoreConfig, layout
    inside, outside, msg = BOUNDS[bound]
    layout(CoreConfig(**inside))
    with pytest.raises(RuntimeError, match=re.escape(msg)):
        layout(CoreConfig(**outside))
