"""SacCore: thin Python object over one libb200sac handle (R co-scheduled learners).

Host-side plumbing only -- torch is used for device buffers / streams; all math
runs in the CUDA library.  The reference-shaped `Learner` classes
(distributed_sac_b200/learner.py) are built on this.
"""
import ctypes as C
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional

import numpy as np
import torch

from . import _lib


@dataclass
class CoreConfig:
    state_dim: int = 8
    act_dim: int = 2
    actor_hidden: List[int] = field(default_factory=lambda: [256, 256])
    critic_hidden: List[int] = field(default_factory=lambda: [256, 256])
    batch: int = 256
    num_tasks: int = 0
    weighted_loss: bool = False
    replicas: int = 1
    precision: int = 0
    gamma: float = 0.99
    tau: float = 0.005
    reward_scale: float = 1.0
    lr_actor: float = 3e-4
    lr_critic: float = 3e-4
    lr_alpha: Optional[float] = None      # the reference uses lr_actor (LL/learner.py:124)
    action_scale: float = 1.0
    beta1: float = 0.9
    beta2: float = 0.999
    adam_eps: float = 1e-8
    log_alpha_init: float = 0.0
    # CARE(M) state encoders (cfg "encoder" block of MT10_Distributed_CARE_cfg.json)
    care: bool = False
    num_encoders: int = 6
    mix_hidden: List[int] = field(default_factory=lambda: [50])
    mix_out: int = 50
    ctx_in: int = 768
    ctx_hidden: List[int] = field(default_factory=lambda: [50, 50])
    ctx_out: int = 50
    tau_se: float = 0.05
    care_original: bool = False          # CARE(O): trainable context encoder (use_modified_care: false)
    emb_dim: int = 50
    lr_ctx: float = 3e-4
    grad_clip: bool = False              # the step plan with gradient-norm clipping and norms (SacCore.set_grad_clip)
    pcgrad: bool = False                 # the per-layer plan with PCGrad gradient surgery (SacCore.set_pcgrad); num_tasks >= 2
    critic_layer_norm: bool = False      # LayerNorm between every hidden Linear and its ReLU in q1, q2 and their targets
    critic_dropout: bool = False         # with critic_layer_norm: dropout before every critic LayerNorm (SacCore.set_critic_dropout)
    critic_ensemble: int = 0             # 0: twin critics; E in [2, 10]: critics q1 .. qE with a target subset (SacCore.set_ensemble)

    @property
    def obs_dim(self):
        return self.state_dim + self.num_tasks

    def to_c(self):
        c = _lib.Cfg()
        c.state_dim, c.act_dim, c.num_tasks = self.state_dim, self.act_dim, self.num_tasks
        c.n_actor_hidden, c.n_critic_hidden = len(self.actor_hidden), len(self.critic_hidden)
        if max(c.n_actor_hidden, c.n_critic_hidden) > _lib.MAX_HIDDEN:
            raise ValueError(f"at most {_lib.MAX_HIDDEN} hidden layers")
        for i, v in enumerate(self.actor_hidden):
            c.actor_hidden[i] = int(v)
        for i, v in enumerate(self.critic_hidden):
            c.critic_hidden[i] = int(v)
        c.batch, c.weighted_loss, c.replicas, c.precision = self.batch, int(self.weighted_loss), self.replicas, self.precision
        c.gamma, c.tau, c.reward_scale = self.gamma, self.tau, self.reward_scale
        c.lr_actor, c.lr_critic = self.lr_actor, self.lr_critic
        c.lr_alpha = self.lr_actor if self.lr_alpha is None else self.lr_alpha
        c.action_scale = self.action_scale
        c.beta1, c.beta2, c.adam_eps = self.beta1, self.beta2, self.adam_eps
        c.log_alpha_init = self.log_alpha_init
        c.care = (2 if self.care_original else 1) if self.care else 0
        c.grad_clip = int(self.grad_clip)
        c.pcgrad = int(self.pcgrad)
        c.critic_ln = int(self.critic_layer_norm)
        c.critic_dropout = int(self.critic_dropout)
        c.critic_ensemble = int(self.critic_ensemble)
        if self.care:
            c.emb_dim, c.lr_ctx = self.emb_dim, self.lr_ctx
            c.num_encoders, c.mix_out, c.ctx_in, c.ctx_out = self.num_encoders, self.mix_out, self.ctx_in, self.ctx_out
            c.n_mix_hidden, c.n_ctx_hidden = len(self.mix_hidden), len(self.ctx_hidden)
            for i, v in enumerate(self.mix_hidden):
                c.mix_hidden[i] = int(v)
            for i, v in enumerate(self.ctx_hidden):
                c.ctx_hidden[i] = int(v)
            c.tau_se = self.tau_se
        return c


def layout(cfg: CoreConfig):
    """Parameter layout table from the C library (pure host call, works without a GPU).
    Returns ({name: (offset, rows, cols, trainable, opt)}, arena_floats, trainable_floats)."""
    lib = _lib.load()
    c = cfg.to_c()
    n, arena, train = C.c_int32(0), C.c_int64(0), C.c_int64(0)
    _lib.check(lib.b200sac_layout(C.byref(c), None, 0, C.byref(n), C.byref(arena), C.byref(train)))
    descs = (_lib.TensorDesc * n.value)()
    _lib.check(lib.b200sac_layout(C.byref(c), descs, n.value, C.byref(n), C.byref(arena), C.byref(train)))
    table = {d.name.decode(): (d.offset, d.rows, d.cols, d.trainable, d.opt, d.pitch) for d in descs}
    return table, arena.value, train.value


def _ptr(t):
    return C.c_void_p(t.data_ptr()) if t is not None else C.c_void_p(0)


_raw_stream = getattr(torch._C, "_cuda_getCurrentRawStream", None)


def _stream():
    """torch's current stream as a cudaStream_t (the raw-stream query skips building a torch.cuda.Stream object: ~2 us per call
    saved on the per-update path)."""
    if _raw_stream is not None:
        return C.c_void_p(_raw_stream(torch.cuda.current_device()))
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _replicas(n, replica):
    """The replicas a per-replica setter writes: `replica`, or all n of them when it is None."""
    return range(n) if replica is None else [int(replica)]


ENSEMBLE_ACTOR = ("min", "mean")     # the actor's reduction over a critic ensemble, by its b200sac_set_ensemble code
RESET_PARTS = ("actor", "critic", "alpha", "encoder", "context")      # index of b200sac_reset_spec.part[]


def reset_parts(cfg: CoreConfig):
    """The parts a b200sac_reset of a handle with this config can touch."""
    return RESET_PARTS[:3] + ((("encoder", "context") if cfg.care_original else ("encoder",)) if cfg.care else ())


def reset_spec(cfg: CoreConfig, shrink=0.0, **parts):
    """The b200sac_reset_spec of SacCore.reset's keywords (pure host function).  actor / critic: a Linear layer count
    from the output layer (0 = untouched) or "all"; alpha / encoder / context: a bool; with no part given, every part the
    handle has.  shrink: one lambda in [0, 1] for every part, or {part: lambda} (parts left out: 0).  Raises ValueError."""
    unknown = set(parts) - set(RESET_PARTS)
    if unknown:
        raise ValueError(f"unknown reset parts {sorted(unknown)}; parts: {RESET_PARTS}")
    given = dict(parts)
    if all(v is None for v in given.values()):
        given = {k: ("all" if k in ("actor", "critic") else True) for k in reset_parts(cfg)}
    have = reset_parts(cfg)
    if isinstance(shrink, dict):
        unknown = set(shrink) - set(RESET_PARTS)
        if unknown:
            raise ValueError(f"shrink names unknown parts {sorted(unknown)}; parts: {RESET_PARTS}")
        lam = {k: shrink.get(k, 0.0) for k in RESET_PARTS}
    else:
        lam = {k: shrink for k in RESET_PARTS}
    spec = _lib.ResetSpec()
    for i, k in enumerate(RESET_PARTS):
        v, x = given.get(k), lam[k]
        if isinstance(x, bool) or not isinstance(x, (int, float, np.integer, np.floating)) or not 0.0 <= float(x) <= 1.0:
            raise ValueError(f"shrink of {k} must be a number in [0, 1], got {x!r}")
        spec.part[i].shrink = float(x)
        if v is None:
            continue
        if k in ("actor", "critic"):
            if v == "all":
                v = len(cfg.actor_hidden if k == "actor" else cfg.critic_hidden) + 1
            if isinstance(v, bool) or not isinstance(v, (int, np.integer)) or v < 0:
                raise ValueError(f"{k} takes a Linear layer count >= 0 or 'all', got {v!r}")
        elif not isinstance(v, (bool, np.bool_)) and not (isinstance(v, (int, np.integer)) and v in (0, 1)):
            raise ValueError(f"{k} takes a bool, got {v!r}")
        if v and k not in have:
            raise ValueError(f"this handle has no {k} to reset (parts: {have})")
        spec.part[i].layers = int(v)
    return spec


REDO_NETS = ("actor", "q1", "q2")        # the order of b200sac_redo's record


def redo_taus(actor=None, critic=None):
    """(tau_actor, tau_critic) of SacCore.redo's keywords (pure host function).  A threshold tau: neurons whose score is
    <= tau are recycled; None = score only (-inf: a negative tau recycles nothing).  Raises ValueError on anything that is
    not a number and on NaN."""
    out = []
    for k, v in (("actor", actor), ("critic", critic)):
        if v is None:
            out.append(-math.inf)
            continue
        if isinstance(v, (bool, np.bool_)) or not isinstance(v, (int, float, np.integer, np.floating)) or math.isnan(float(v)):
            raise ValueError(f"{k} takes a dormancy threshold (a number, not NaN) or None, got {v!r}")
        out.append(float(v))
    return tuple(out)


class SacCore:
    def __init__(self, cfg: CoreConfig, device: int = 0, seed: int = 0):
        self.lib = _lib.load()
        if not torch.cuda.is_available():
            raise RuntimeError("SacCore needs a CUDA device (sm_90a); there is no CPU fallback")
        self.cfg = cfg
        self.device = torch.device("cuda", device)
        self.table, self.arena_floats, self.trainable_floats = layout(cfg)
        self._h = C.c_void_p(0)
        c = cfg.to_c()
        torch.cuda.set_device(self.device)
        _lib.check(self.lib.b200sac_create(C.byref(c), device, C.c_uint64(seed), C.byref(self._h)))
        n = C.c_int32(0)
        _lib.check(self.lib.b200sac_launches_per_step(self._h, C.byref(n)))
        self.launches_per_step = n.value
        self.steps_done = 0
        self._loss_buf = (C.c_float * (4 * max(1, cfg.replicas)))()

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value:
            self.lib.b200sac_destroy(self._h)
            self._h = C.c_void_p(0)

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # ---- state ------------------------------------------------------------------------
    def _arena_n(self, which):
        return self.arena_floats if which == _lib.PARAMS else self.trainable_floats

    def export_arena(self, which=_lib.PARAMS, replica=0) -> torch.Tensor:
        out = torch.empty(self._arena_n(which), dtype=torch.float32)
        _lib.check(self.lib.b200sac_export(self._h, which, replica, _ptr(out), out.numel(), _stream()))
        return out

    def import_arena(self, flat: torch.Tensor, which=_lib.PARAMS, replica=0):
        flat = flat.detach().to(torch.float32).contiguous()
        assert flat.numel() == self._arena_n(which)
        _lib.check(self.lib.b200sac_import(self._h, which, replica, _ptr(flat), flat.numel(), _stream()))

    def arena_view(self, which=_lib.PARAMS):
        """(device pointer, floats per replica) of an arena (replicas contiguous)."""
        p, n = C.c_void_p(0), C.c_int64(0)
        _lib.check(self.lib.b200sac_arena_ptr(self._h, which, C.byref(p), C.byref(n)))
        return p.value, n.value

    def _unpack(self, name, flat, off):
        """One layout-table entry read out of `flat` (float32 numpy array) at float offset `off`, as a fresh CPU tensor in
        the reference's shape.  numpy copies on purpose: a 256x256 torch .clone() fans out to the intra-op thread pool,
        which costs milliseconds on a busy host."""
        return torch.from_numpy(np.array(self._view(name, flat, off), dtype=np.float32, order="C", copy=True))

    def _view(self, name, flat, off):
        """numpy view (no copy) of one layout-table entry inside `flat`, in the reference's shape."""
        _, rows, cols, _t, _o, pitch = self.table[name]
        a = flat[off:off + rows * pitch].reshape(rows, pitch)[:, :cols]
        if ".mix." in name:            # stored as [K][out][in] | [K][out]; the reference holds (K,in,out) | (K,1,out)
            K = self.cfg.num_encoders
            a = (a.reshape(K, rows // K, cols).transpose(0, 2, 1) if name.endswith(".W") else a.reshape(K, 1, rows // K))
        elif not (name.endswith(".weight") or name == "embedding"):
            a = a.reshape(-1)
        return a

    def act(self, obs, stochastic=True, eps=None, replica=0, no_tanh=False) -> torch.Tensor:
        """Batched Actor.get_action for n <= 2*batch (CARE: batch) observation rows (CPU or CUDA tensor [n][obs_dim]); returns a
        CPU tensor [n][act_dim].  eps ([n][act_dim]) injects the noise; stochastic=False gives k*tanh(mu), or k*mu with
        no_tanh=True (the LunarLander actor's deterministic action)."""
        obs = obs.to(torch.float32).contiguous()
        n = obs.shape[0]
        e = None if eps is None else eps.to(torch.float32).contiguous()
        out = torch.empty(n, self.cfg.act_dim)
        _lib.check(self.lib.b200sac_act(self._h, replica, n, _ptr(obs), _ptr(e), 1 if stochastic else (-1 if no_tanh else 0), _ptr(out), _stream()))
        return out

    def critic_values(self, obs, act, target=False, replica=0):
        """(q1, q2) of one replica on n >= 1 rows obs [n][obs_dim] and act [n][act_dim] (CPU or CUDA tensors), or of
        q1_target and q2_target with target=True: two [n] tensors on the device obs is on; on a critic_ensemble handle one
        [E][n] tensor of q1 .. qE (or their targets).  Eval mode (no dropout), any n, every row's values independent of the
        others (b200sac_critic_values).  Synchronises the current stream."""
        if not isinstance(target, (bool, np.bool_)):
            raise ValueError(f"target must be a bool, got {target!r}")
        obs = torch.as_tensor(obs).to(torch.float32).contiguous()
        act = torch.as_tensor(act).to(obs.device, torch.float32).contiguous()
        n = obs.shape[0] if obs.dim() == 2 else 0
        if n < 1 or obs.shape != (n, self.cfg.obs_dim) or act.shape != (n, self.cfg.act_dim):
            raise ValueError(f"obs must be [n][{self.cfg.obs_dim}] and act [n][{self.cfg.act_dim}] with n >= 1, got "
                             f"{tuple(obs.shape)} and {tuple(act.shape)}")
        out = torch.empty(self.n_critics, n, device=obs.device)
        _lib.check(self.lib.b200sac_critic_values(self._h, int(replica), n, _ptr(obs), _ptr(act), 1 if target else 0, _ptr(out),
                                                  _stream()))
        return out if self.cfg.critic_ensemble else (out[0], out[1])

    @property
    def n_critics(self) -> int:
        """Critics per replica: cfg.critic_ensemble, or 2 (the twins)."""
        return int(self.cfg.critic_ensemble) or 2

    def critic_values_chunk(self) -> int:
        """Rows critic_values and Replay.refresh_priorities evaluate per launch sequence (their scratch holds that many)."""
        n = C.c_int64(0)
        _lib.check(self.lib.b200sac_critic_values_chunk(self._h, C.byref(n)))
        return n.value

    def read_named(self, name, which=_lib.PARAMS, replica=0) -> torch.Tensor:
        """One small tensor (e.g. log_alpha) straight from the device: a few floats cross PCIe, not the arena."""
        off, rows, cols, _t, _o, pitch = self.table[name]
        out = torch.empty(rows * pitch)
        _lib.check(self.lib.b200sac_read_range(self._h, which, replica, off, rows * pitch, _ptr(out), _stream()))
        return self._unpack(name, out.numpy(), 0)

    # ---- blob publication (b200sac_blob_*): the published byte string is assembled on the device -------------------
    def tensor_shape(self, name):
        """Shape of tensor `name` as the reference's state_dict holds it."""
        off, rows, _cols, _t, _o, pitch = self.table[name]
        return tuple(self._view(name, np.broadcast_to(np.float32(0), (off + rows * pitch,)), off).shape)

    def blob_index_map(self, name) -> np.ndarray:
        """Arena index of every element of tensor `name`, in the reference's shape and C order (pitch padding and the
        CARE mixture transposition are resolved here, once)."""
        off, rows, _cols, _t, _o, pitch = self.table[name]
        idx = np.arange(off + rows * pitch, dtype=np.int64)
        return np.ascontiguousarray(self._view(name, idx, off)).reshape(-1)

    def blob_template(self, image: bytes, slots, extra=(), replica=0):
        """Register the byte image.  slots: [(tensor name, byte offset of its payload inside `image`)]; extra: tensor names
        whose floats are appended BEHIND the image bytes (4-byte aligned; e.g. log_alpha for the logger) and returned by
        blob_wait() as numpy arrays."""
        src, dst = [], []
        for name, at in slots:
            m = self.blob_index_map(name)
            src.append(m)
            dst.append(at + 4 * np.arange(m.size, dtype=np.int64))
        total = (len(image) + 3) & ~3
        self._blob_extra = []
        for name in extra:
            m = self.blob_index_map(name)
            src.append(m)
            dst.append(total + 4 * np.arange(m.size, dtype=np.int64))
            self._blob_extra.append((name, total, m.size))
            total += 4 * m.size
        src = np.ascontiguousarray(np.concatenate(src), dtype=np.int32)
        dst = np.ascontiguousarray(np.concatenate(dst), dtype=np.int32)
        img = np.zeros(total, dtype=np.uint8)
        img[:len(image)] = np.frombuffer(image, dtype=np.uint8)
        _lib.check(self.lib.b200sac_blob_template(self._h, replica, C.c_void_p(img.ctypes.data), total, src.size,
                                                  C.c_void_p(src.ctypes.data), C.c_void_p(dst.ctypes.data)))
        self._blob_len = len(image)

    def blob_begin(self):
        _lib.check(self.lib.b200sac_blob_begin(self._h, _stream()))

    def blob_wait(self):
        """(published bytes, {extra tensor name: float32 array}) of the oldest blob begun and not yet collected."""
        ptr, n = C.c_void_p(), C.c_int64()
        _lib.check(self.lib.b200sac_blob_wait(self._h, C.byref(ptr), C.byref(n)))
        blob = C.string_at(ptr.value, self._blob_len)
        extra = {name: np.ctypeslib.as_array(C.cast(ptr.value + at, C.POINTER(C.c_float)), shape=(cnt,)).copy()
                 for name, at, cnt in self._blob_extra}
        return blob, extra

    def get_named(self, which=_lib.PARAMS, replica=0) -> Dict[str, torch.Tensor]:
        flat = self.export_arena(which, replica).numpy()
        return {name: self._unpack(name, flat, d[0]) for name, d in self.table.items() if which == _lib.PARAMS or d[3]}

    def set_named(self, tensors: Dict[str, torch.Tensor], which=_lib.PARAMS, replica=0, strict=True):
        flat = self.export_arena(which, replica)
        seen = set()
        for name, t in tensors.items():
            if name not in self.table:
                if strict:
                    raise KeyError(name)
                continue
            off, rows, cols, trainable, _, pitch = self.table[name]
            if which != _lib.PARAMS and not trainable:
                continue
            t = torch.as_tensor(t, dtype=torch.float32)
            if ".mix." in name and name.endswith(".W"):
                t = t.permute(0, 2, 1).contiguous()          # (K,in,out) -> [K][out][in]
            t = t.reshape(-1)
            if t.numel() != rows * cols:
                raise ValueError(f"{name}: expected {rows * cols} elements, got {t.numel()}")
            flat[off:off + rows * pitch].reshape(rows, pitch)[:, :cols] = t.reshape(rows, cols)
            seen.add(name)
        if strict:
            need = {n for n, d in self.table.items() if which == _lib.PARAMS or d[3]}
            if need - seen:
                raise KeyError(f"missing tensors: {sorted(need - seen)[:5]}")
        self.import_arena(flat, which, replica)

    def get_steps(self, replica=0):
        s = (C.c_int64 * 4)()
        _lib.check(self.lib.b200sac_get_steps(self._h, replica, s))
        n = 4 if (self.cfg.care and self.cfg.care_original) else 3
        return tuple(int(x) for x in s)[:n]     # (critic, actor, alpha[, context encoder])

    def set_steps(self, steps, replica=0):
        cur = list(self.get_steps(replica)) + [0]
        vals = [int(x) for x in steps] + cur[len(steps):4]
        s = (C.c_int64 * 4)(*vals[:4])
        _lib.check(self.lib.b200sac_set_steps(self._h, replica, s))

    # ---- per-replica hyperparameters (b200sac_get/set_hparams) -------------------------------------------
    HPARAMS = tuple(name for name, _ in _lib.Hparams._fields_)

    def get_hparams(self, replica=0) -> Dict[str, float]:
        """{gamma, reward_scale, tau, lr_critic, lr_actor, lr_alpha, tau_se, lr_ctx} of one replica (no synchronisation)."""
        hp = _lib.Hparams()
        _lib.check(self.lib.b200sac_get_hparams(self._h, int(replica), C.byref(hp)))
        return {name: float(getattr(hp, name)) for name in self.HPARAMS}

    def set_hparams(self, replica=None, **values):
        """Change hyperparameters of one replica (replica=None: all of them) on the current stream; fields not named keep
        their value.  Steps enqueued afterwards use the new values, steps already enqueued do not."""
        unknown = set(values) - set(self.HPARAMS)
        if unknown:
            raise TypeError(f"unknown hyperparameters {sorted(unknown)}; known: {self.HPARAMS}")
        for r in _replicas(self.cfg.replicas, replica):
            cur = self.get_hparams(r)
            cur.update({k: float(v) for k, v in values.items()})
            hp = _lib.Hparams(**cur)
            _lib.check(self.lib.b200sac_set_hparams(self._h, r, C.byref(hp), _stream()))

    # ---- per-replica update intervals (b200sac_get/set_update_intervals) -------------------------------------
    def get_update_intervals(self, replica=0):
        """(actor_every, target_every) of one replica (no synchronisation)."""
        a, t = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.b200sac_get_update_intervals(self._h, int(replica), C.byref(a), C.byref(t)))
        return a.value, t.value

    def set_update_intervals(self, actor_every=None, target_every=None, replica=None):
        """Update the actor (and temperature) only on steps whose critic step count n is a multiple of actor_every, and the
        targets only when n is a multiple of target_every, for one replica (replica=None: all of them) on the current
        stream; an interval not named keeps its value.  Steps enqueued afterwards follow the new schedule."""
        for r in _replicas(self.cfg.replicas, replica):
            a, t = self.get_update_intervals(r)
            a = a if actor_every is None else int(actor_every)
            t = t if target_every is None else int(target_every)
            _lib.check(self.lib.b200sac_set_update_intervals(self._h, r, a, t, _stream()))

    # ---- gradient-norm clipping (b200sac_set/get_grad_clip, b200sac_read_grad_norms; handles with grad_clip=True) ------
    CLIP_NAMES = ("critic", "actor", "ctx")

    def get_grad_clip(self, replica=0) -> Dict[str, float]:
        """{critic, actor, ctx} max-norm thresholds of one replica (no synchronisation); inf = no clipping."""
        v = [C.c_double() for _ in self.CLIP_NAMES]
        _lib.check(self.lib.b200sac_get_grad_clip(self._h, int(replica), *[C.byref(x) for x in v]))
        return {k: x.value for k, x in zip(self.CLIP_NAMES, v)}

    def set_grad_clip(self, critic=None, actor=None, ctx=None, replica=None):
        """clip_grad_norm_ thresholds of the critic, actor and CARE(O) context-encoder optimizers of one replica
        (replica=None: all of them) on the current stream; a name left out keeps its value, inf turns clipping off.
        Steps enqueued afterwards use them."""
        for r in _replicas(self.cfg.replicas, replica):
            cur = self.get_grad_clip(r)
            for k, v in dict(critic=critic, actor=actor, ctx=ctx).items():
                if v is not None:
                    cur[k] = float(v)
            _lib.check(self.lib.b200sac_set_grad_clip(self._h, r, cur["critic"], cur["actor"], cur["ctx"], _stream()))

    # ---- critic dropout (b200sac_set/get_critic_dropout; handles with critic_dropout=True) --------------------------------
    def get_critic_dropout(self, replica=0) -> float:
        """The critic dropout rate p of one replica (no synchronisation)."""
        p = C.c_double()
        _lib.check(self.lib.b200sac_get_critic_dropout(self._h, int(replica), C.byref(p)))
        return p.value

    def set_critic_dropout(self, p, replica=None):
        """Dropout rate p in [0, 1) before every critic LayerNorm of one replica (replica=None: all of them), on the current
        stream.  Steps enqueued afterwards use it."""
        for r in _replicas(self.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_set_critic_dropout(self._h, r, float(p), _stream()))

    # ---- critic ensembles (b200sac_set/get_ensemble; handles with critic_ensemble=E) ---------------------------------------
    ENSEMBLE_ACTOR = ENSEMBLE_ACTOR

    def get_ensemble(self, replica=0):
        """(m, actor) of one replica: the target subset size and "mean" or "min" (no synchronisation)."""
        m, mean = C.c_int32(), C.c_int32()
        _lib.check(self.lib.b200sac_get_ensemble(self._h, int(replica), C.byref(m), C.byref(mean)))
        return m.value, self.ENSEMBLE_ACTOR[mean.value]

    def set_ensemble(self, m, actor="mean", replica=None):
        """Target subset size m in [1, E] and the actor's reduction over the E critics ("mean" or "min") of one replica
        (replica=None: all of them), on the current stream.  Steps enqueued afterwards use them."""
        if actor not in self.ENSEMBLE_ACTOR:
            raise ValueError(f"actor must be 'mean' or 'min', got {actor!r}")
        for r in _replicas(self.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_set_ensemble(self._h, r, int(m), self.ENSEMBLE_ACTOR.index(actor), _stream()))

    def read_grad_norms(self, n_last: int = 1) -> torch.Tensor:
        """Pre-clip gradient norms [n_last][R][3] (critic, actor, context encoder) of the last steps, aligned with read_losses;
        NaN where that optimizer did not step."""
        out = torch.empty(n_last, self.cfg.replicas, 3)
        _lib.check(self.lib.b200sac_read_grad_norms(self._h, int(n_last), _ptr(out), _stream()))
        return out

    # ---- PCGrad gradient surgery (b200sac_set/get/read_pcgrad, b200sac_export_task_grad; handles with pcgrad=True) --------
    def get_pcgrad(self, replica=0) -> Dict[str, bool]:
        """{critic, actor} surgery switches of one replica (no synchronisation)."""
        c, a = C.c_int32(0), C.c_int32(0)
        _lib.check(self.lib.b200sac_get_pcgrad(self._h, int(replica), C.byref(c), C.byref(a)))
        return {"critic": bool(c.value), "actor": bool(a.value)}

    def set_pcgrad(self, critic=None, actor=None, replica=None):
        """Turn the critic's / actor's gradient surgery on or off for one replica (replica=None: all of them) on the current
        stream; a switch left out keeps its value.  Off: Adam reads the plain sum of the task gradients, and the Gram matrix
        is still computed.  Steps enqueued afterwards use the new switches."""
        for r in _replicas(self.cfg.replicas, replica):
            cur = self.get_pcgrad(r)
            for k, v in dict(critic=critic, actor=actor).items():
                if v is not None:
                    cur[k] = bool(v)
            _lib.check(self.lib.b200sac_set_pcgrad(self._h, r, int(cur["critic"]), int(cur["actor"]), _stream()))

    def read_pcgrad(self, replica=0) -> Dict[str, np.ndarray]:
        """The last step's surgery record of one replica, index 0 critic and 1 actor: gram [2][T][T] (fp64), w [2][T],
        perm [2][T][T] (row i = the order task i was projected in), projected [2][T][T] bool (task i onto task j), and
        task_mismatch, the rows of the step that were not in task-block order."""
        T = self.cfg.num_tasks
        gram = np.empty((2, T, T), np.float64)
        w = np.empty((2, T), np.float32)
        perm = np.empty((2, T, T), np.int32)
        mask = np.empty((2, T), np.uint64)
        bad = C.c_int32(0)
        _lib.check(self.lib.b200sac_read_pcgrad(self._h, int(replica), gram.ctypes.data, w.ctypes.data, perm.ctypes.data,
                                                mask.ctypes.data, C.byref(bad), _stream()))
        bits = np.uint64(1) << np.arange(T, dtype=np.uint64)
        projected = (mask[:, :, None] & bits[None, None, :]) != 0
        return {"gram": gram, "w": w, "perm": perm, "projected": projected, "task_mismatch": int(bad.value)}

    # ---- CAGrad (b200sac_set/get/read_cagrad; handles with pcgrad=True) ---------------------------------------------
    def get_cagrad(self, replica=0) -> Dict[str, float]:
        """{critic, actor} CAGrad coefficients c of one replica (no synchronisation); 0 = off."""
        c, a = C.c_double(0), C.c_double(0)
        _lib.check(self.lib.b200sac_get_cagrad(self._h, int(replica), C.byref(c), C.byref(a)))
        return {"critic": c.value, "actor": a.value}

    def set_cagrad(self, critic=None, actor=None, replica=None):
        """CAGrad coefficient c of the critic's / actor's optimizer for one replica (replica=None: all of them) on the
        current stream; a value left out keeps its value.  c > 0: Adam reads the CAGrad combination of the task gradients
        whatever the PCGrad switch says; 0 turns CAGrad off.  Steps enqueued afterwards use the new values."""
        for r in _replicas(self.cfg.replicas, replica):
            cur = self.get_cagrad(r)
            for k, v in dict(critic=critic, actor=actor).items():
                if v is not None:
                    cur[k] = float(v)
            _lib.check(self.lib.b200sac_set_cagrad(self._h, r, cur["critic"], cur["actor"], _stream()))

    def read_cagrad(self, replica=0) -> Dict[str, np.ndarray]:
        """The last step's CAGrad record of one replica, index 0 critic and 1 actor: p [2][T] (the dual's weights p*),
        lambda, best (best objective F), first (F at uniform weights), scale (s) [2] fp64, and ibest [2] (the iteration of
        the best F; -1 = CAGrad did not run, -2 = degenerate Gram matrix).  The weights Adam read are read_pcgrad()["w"]."""
        T = self.cfg.num_tasks
        p = np.empty((2, T), np.float64)
        f = {k: np.empty(2, np.float64) for k in ("lambda", "best", "first", "scale")}
        ib = np.empty(2, np.int32)
        _lib.check(self.lib.b200sac_read_cagrad(self._h, int(replica), p.ctypes.data, f["lambda"].ctypes.data,
                                                f["best"].ctypes.data, f["first"].ctypes.data, f["scale"].ctypes.data,
                                                ib.ctypes.data, _stream()))
        return dict(p=p, ibest=ib, **f)

    def export_task_grad(self, task: int, replica=0) -> torch.Tensor:
        """Gradient of the last step over the rows of task `task` alone (the trainable arena, CPU tensor)."""
        out = torch.empty(self.trainable_floats, dtype=torch.float32)
        _lib.check(self.lib.b200sac_export_task_grad(self._h, int(replica), int(task), _ptr(out), out.numel(), _stream()))
        return out

    def copy_replica(self, src: int, dst: int):
        """Replica dst's parameters (targets, log_alpha included), Adam moments and step counters become a copy of src's,
        device to device on the current stream.  Hyperparameters, update intervals, gradient-clipping thresholds, PCGrad
        switches and replay data stay dst's own."""
        _lib.check(self.lib.b200sac_copy_replica(self._h, int(src), int(dst), _stream()))

    def reset(self, seed: int, replica=None, actor=None, critic=None, alpha=None, encoder=None, context=None, shrink=0.0):
        """Re-initialise networks of one replica (replica=None: every replica, one call each) on the current stream:
        theta = shrink * theta + (1 - shrink) * theta0, theta0 the draw b200sac_create(seed) made, targets alike; the
        owning optimizers restart.  actor / critic: Linear layers from the output ("all" = every layer); alpha, encoder
        (CARE state encoder), context (CARE(O) context encoder): bools; no part given = every part the handle has (a full
        reset).  shrink: a float or {part: float}.  Steps enqueued afterwards see the reset (include/b200sac.h)."""
        spec = reset_spec(self.cfg, shrink, actor=actor, critic=critic, alpha=alpha, encoder=encoder, context=context)
        for r in _replicas(self.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_reset(self._h, r, C.byref(spec), C.c_uint64(int(seed) % (1 << 64)), _stream()))

    def redo(self, seed: int, obs, act, actor=None, critic=None, replica=None):
        """Dormant-neuron recycling (ReDo) of one replica (replica=None: every replica, each under its own key seed +
        replica) on the current stream.  Scores every hidden neuron of the actor, q1 and q2 on the rows obs [n][obs_dim]
        and act [n][act_dim] (1 <= n <= batch, CPU or CUDA), then recycles those whose score is <= the network's threshold:
        actor= for the actor, critic= for q1 and q2; None = score only.  Recycled rows take b200sac_create(seed)'s draw,
        their biases and outgoing weights and the Adam moments there become 0 (include/b200sac.h).  read_redo() shows the
        record; steps enqueued afterwards see the recycled networks."""
        ta, tc = redo_taus(actor, critic)
        obs = obs.to(torch.float32).contiguous()
        act = act.to(torch.float32).contiguous()
        n = obs.shape[0]
        if obs.shape != (n, self.cfg.obs_dim) or act.shape != (n, self.cfg.act_dim):
            raise ValueError(f"obs must be [n][{self.cfg.obs_dim}] and act [n][{self.cfg.act_dim}], got {tuple(obs.shape)} "
                             f"and {tuple(act.shape)}")
        for r in _replicas(self.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_redo(self._h, r, n, _ptr(obs), _ptr(act), ta, tc, C.c_uint64(int(seed) % (1 << 64)),
                                             _stream()))

    def read_redo(self, replica=0) -> Dict[str, Dict[str, List[np.ndarray]]]:
        """The last redo() record of one replica: {"actor" | "q1" | "q2": {"score": [fp64 per hidden layer], "dormant":
        [bool per hidden layer]}}; NaN scores and no dormant neuron before the first call."""
        n = C.c_int64(0)
        _lib.check(self.lib.b200sac_read_redo(self._h, int(replica), None, None, 0, C.byref(n), _stream()))
        score, flag = np.empty(n.value, np.float64), np.empty(n.value, np.uint8)
        _lib.check(self.lib.b200sac_read_redo(self._h, int(replica), C.c_void_p(score.ctypes.data),
                                              C.c_void_p(flag.ctypes.data), n.value, C.byref(n), _stream()))
        out, i = {}, 0
        for net in REDO_NETS:
            widths = self.cfg.actor_hidden if net == "actor" else self.cfg.critic_hidden
            out[net] = {"score": [], "dormant": []}
            for H in widths:
                out[net]["score"].append(score[i:i + H])
                out[net]["dormant"].append(flag[i:i + H].astype(bool))
                i += H
        return out

    def soft_update(self, tau: float, critic: Optional[int] = None):
        """Polyak update of the targets outside a step: both critics (CARE: and the target state encoder, with the replica's
        tau_se unless tau == 1), or with critic=k only q<k>_target (k in [1, 2], or [1, E] on a critic_ensemble handle)."""
        if critic is None:
            _lib.check(self.lib.b200sac_soft_update(self._h, float(tau), _stream()))
        else:
            _lib.check(self.lib.b200sac_soft_update_critic(self._h, int(critic), float(tau), _stream()))

    # ---- stepping -----------------------------------------------------------------------
    def _shape_check(self, s, a, r, s2, d, eps_next, eps_cur):
        c = self.cfg
        R, B = c.replicas, c.batch
        want = dict(s=c.obs_dim, a=c.act_dim, r=1, s2=c.obs_dim, d=1)
        for k, t in dict(s=s, a=a, r=r, s2=s2, d=d).items():
            if t.numel() != R * B * want[k]:
                raise ValueError(f"{k}: expected {R}x{B}x{want[k]} elements, got {tuple(t.shape)}")
        for k, t in dict(eps_next=eps_next, eps_cur=eps_cur).items():
            if t is not None and t.numel() != R * B * c.act_dim:
                raise ValueError(f"{k}: expected {R}x{B}x{c.act_dim} elements, got {tuple(t.shape)}")

    def step(self, s, a, r, s2, d, eps_next=None, eps_cur=None):
        """One gradient step from DEVICE tensors [R][B][w] (asynchronous)."""
        ts = [None if t is None else t.to(self.device, torch.float32).contiguous() for t in (s, a, r, s2, d, eps_next, eps_cur)]
        self._shape_check(*ts)
        self._keep = ts          # keep inputs alive until the stream has consumed them
        _lib.check(self.lib.b200sac_step(self._h, *[_ptr(t) for t in ts], _stream()))
        self.steps_done += 1

    def step_host(self, s, a, r, s2, d, eps_next=None, eps_cur=None, want_losses=True):
        """One gradient step from HOST tensors through the pinned staging path; returns
        losses [R][4] = (critic, actor, alpha, entropy) if want_losses (synchronises)."""
        ts = [None if t is None else t.detach().to("cpu", torch.float32).contiguous() for t in (s, a, r, s2, d, eps_next, eps_cur)]
        self._shape_check(*ts)
        out = torch.empty(self.cfg.replicas, 4) if want_losses else None
        _lib.check(self.lib.b200sac_step_host(self._h, *[_ptr(t) for t in ts], _ptr(out), _stream()))
        self.steps_done += 1
        return out

    def step_sampled(self, replay: "Replay", n_steps: int = 1):
        _lib.check(self.lib.b200sac_step_sampled(self._h, replay._h, int(n_steps), _stream()))
        self.steps_done += int(n_steps)

    def prepare(self, replay: "Replay"):
        """Instantiate every CUDA graph the sampled path can launch for this ring (no step is run)."""
        _lib.check(self.lib.b200sac_prepare(self._h, replay._h, _stream()))

    def update_sampled(self, replay: "Replay"):
        """sample + one gradient step + that step's losses of replica 0 as python floats (critic, actor, alpha, entropy):
        one library call, no tensor round trips -- the body of Learner.update()."""
        buf = self._loss_buf
        _lib.check(self.lib.b200sac_update(self._h, replay._h, buf, _stream()))
        self.steps_done += 1
        return buf[0], buf[1], buf[2], buf[3]

    def read_losses(self, n_last: int = 1) -> torch.Tensor:
        out = torch.empty(n_last, self.cfg.replicas, 4)
        _lib.check(self.lib.b200sac_read_losses(self._h, n_last, _ptr(out), _stream()))
        return out

    def profile_step(self, replay: "Replay", iters: int = 20):
        """[(kernel label, mean ms)] per launch of one step (eager run with CUDA events)."""
        cap = 256
        out = (C.c_float * cap)()
        n = C.c_int32(0)
        names = C.create_string_buffer(8192)
        _lib.check(self.lib.b200sac_profile_step(self._h, replay._h, int(iters), out, cap, C.byref(n), names, 8192, _stream()))
        self.steps_done += int(iters)
        labels = names.value.decode().split(";")
        return [(labels[i], float(out[i])) for i in range(n.value)]

    def graph_timeline(self, replay: "Replay", iters: int = 200):
        """Mean in-graph start-to-start time (us) of every launch of one step: [sample, ingest, plan...]."""
        cap = 256
        out = (C.c_float * cap)()
        n = C.c_int32(0)
        _lib.check(self.lib.b200sac_graph_timeline(self._h, replay._h, int(iters), out, cap, C.byref(n), _stream()))
        self.steps_done += int(iters) + 6
        return [float(out[i]) for i in range(n.value)]

    def debug(self, name: str, replica=0) -> torch.Tensor:
        """Per-step intermediates (b200sac_debug_read): y, q1, ..., and the hidden activations "hA.<l>", "hQ.<l>", "hP.<l>",
        "hT.<l>", "mixH.<inst>.<l>" whose sign patterns are the ReLU masks the step used; with critic_layer_norm, "zQ.<l>",
        "zP.<l>", "zT.<l>" before the normalization (after the dropout with critic_dropout); with critic_dropout, "mQ.<l>",
        "mP.<l>", "mT.<l>" the keep masks (0.0 / 1.0).  After a step from a prioritized
        ring: "isw" (importance weights), "prio" (leaf values written) and "idx" (ring indices, int32).  After a step from a
        ring with trajectory links: "disc" (per-row discount), "nstep_m" (hops folded, int32), "idx"; "r" and "d" are folded."""
        cap = self.cfg.batch * max(2 * self.cfg.act_dim, 1)
        if name in ("idx", "nstep_m"):          # int32: ring indices (prioritized / linked ring), hops folded (linked ring)
            return self._debug_raw(name, replica, cap).view(torch.int32)
        if name == "psave":
            cap = 2 * self.cfg.batch * self.cfg.act_dim * 8
        elif name == "head":
            cap = 2 * self.cfg.batch * 2 * self.cfg.act_dim
        elif name[0] in "hzm":
            widest = max(list(self.cfg.actor_hidden) + list(self.cfg.critic_hidden) + [4 * ((w + 3) // 4) * self.cfg.num_encoders
                                                                                        for w in self.cfg.mix_hidden])
            cap = max(2, self.n_critics) * self.cfg.batch * widest
        elif name in ("q_pi", "dq_pi"):
            cap = self.n_critics * self.cfg.batch
        return self._debug_raw(name, replica, cap)

    def _debug_raw(self, name, replica, cap):
        out = torch.empty(cap)
        n = C.c_int64(0)
        _lib.check(self.lib.b200sac_debug_read(self._h, name.encode(), replica, _ptr(out), cap, C.byref(n), _stream()))
        return out[:n.value].clone()


class Replay:
    """Replay ring in HBM (where='device') or pinned host DRAM (where='host').

    prioritized=dict(alpha=, beta=, eps=) makes a prioritized device ring (sum-tree sampling, importance-weighted critic
    loss, priorities updated inside every step; see include/b200sac.h).  trajectories=True keeps trajectory links on the
    device ring, so that steps can train on n-step returns (set_nstep)."""

    def __init__(self, core: SacCore, capacity: int, where: str = "device", seed: int = 0, prioritized=None, trajectories=False):
        self.core = core
        self.lib = core.lib
        self._h = C.c_void_p(0)
        self._prior = None
        self.capacity = int(capacity)
        w = {"device": 0, "host": 1}[where]
        self.prioritized = None if prioritized is None else dict(prioritized)
        if self.prioritized is not None:
            if where != "device":
                raise ValueError("prioritized replay needs the device ring (where='device')")
            unknown = set(self.prioritized) - {"alpha", "beta", "eps"}
            if unknown or len(self.prioritized) != 3:
                raise ValueError(f"prioritized= takes exactly alpha, beta and eps (got {sorted(self.prioritized)})")
            p = self.prioritized
            _lib.check(self.lib.b200sac_replay_create_prioritized(core._h, int(capacity), C.c_uint64(seed), float(p["alpha"]),
                                                                  float(p["beta"]), float(p["eps"]), C.byref(self._h)))
        else:
            _lib.check(self.lib.b200sac_replay_create(core._h, int(capacity), w, C.c_uint64(seed), C.byref(self._h)))
        self.where = where
        self.trajectories = bool(trajectories)
        if self.trajectories:
            if where != "device":
                self.close()
                raise ValueError("trajectory links (n-step returns) need the device ring (where='device')")
            _lib.check(self.lib.b200sac_replay_enable_trajectories(self._h))

    def close(self):
        if getattr(self, "_h", None) is not None and self._h.value and self.core._h.value:
            self.lib.b200sac_replay_destroy(self._h)         # (detaches the prior first, or from the ring it is the prior of)
        self._h = C.c_void_p(0)
        self._prior = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def push(self, s, a, r, s2, d, replica=0, stream=None, cut=None):
        """Append rows.  stream (scalar or one id per row, in [0, 65536)) says which player / environment each row came from,
        so that a ring with trajectory links can chain consecutive rows of a stream; cut (scalar or per row) marks a
        time-limit truncation.  stream=None is the plain push (the rows join no trajectory)."""
        ts = [np.ascontiguousarray(np.asarray(t, dtype=np.float32)) for t in (s, a, r, s2, d)]
        n = ts[2].size
        if stream is None:
            if cut is not None:
                raise ValueError("cut= needs stream=")
            _lib.check(self.lib.b200sac_replay_push(self._h, replica, n, *[C.c_void_p(t.ctypes.data) for t in ts]))
            return
        sid = np.ascontiguousarray(np.broadcast_to(np.asarray(stream, dtype=np.int32).reshape(-1), (n,)))
        ct = None if cut is None else np.ascontiguousarray(np.broadcast_to(np.asarray(cut).astype(np.uint8).reshape(-1), (n,)))
        _lib.check(self.lib.b200sac_replay_push_traj(self._h, replica, n, *[C.c_void_p(t.ctypes.data) for t in ts],
                                                     C.c_void_p(sid.ctypes.data), C.c_void_p(0 if ct is None else ct.ctypes.data)))

    def fill_synthetic(self, n: int, seed: int = 1234):
        _lib.check(self.lib.b200sac_replay_fill_synthetic(self._h, int(n), C.c_uint64(seed), _stream()))

    def size(self, replica=0) -> int:
        n = C.c_int64(0)
        _lib.check(self.lib.b200sac_replay_size(self._h, replica, C.byref(n)))
        return n.value

    def sample(self, replica=0, with_indices=False):
        c = self.core.cfg
        B = c.batch
        s, a, r = torch.empty(B, c.obs_dim), torch.empty(B, c.act_dim), torch.empty(B, 1)
        s2, d = torch.empty(B, c.obs_dim), torch.empty(B, 1)
        idx = torch.empty(B, dtype=torch.int64)
        _lib.check(self.lib.b200sac_replay_sample(self._h, replica, _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d), _ptr(idx)))
        return (s, a, r, s2, d, idx) if with_indices else (s, a, r, s2, d)

    # ---- prioritized replay -----------------------------------------------------------------
    def set_beta(self, beta: float, replica=None):
        """Importance-sampling exponent of one replica (None: all), in stream order: steps enqueued afterwards use it."""
        for r in _replicas(self.core.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_replay_set_beta(self._h, r, float(beta), _stream()))

    def set_priorities(self, idx, prio, replica=0):
        """Raw priorities (>= 0; (prio + eps)^alpha is stored) of filled ring slots `idx`; a later entry wins a duplicate."""
        idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1))
        prio = np.ascontiguousarray(np.asarray(prio, dtype=np.float32).reshape(-1))
        if idx.size != prio.size:
            raise ValueError("idx and prio differ in length")
        _lib.check(self.lib.b200sac_replay_set_priorities(self._h, int(replica), idx.size, C.c_void_p(idx.ctypes.data),
                                                          C.c_void_p(prio.ctypes.data)))

    def priorities(self, idx, replica=0) -> np.ndarray:
        """Leaf values p of ring slots `idx` (an index -1 - t gives task t's root sum)."""
        idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1))
        out = np.empty(idx.size, dtype=np.float32)
        _lib.check(self.lib.b200sac_replay_get_priorities(self._h, int(replica), idx.size, C.c_void_p(idx.ctypes.data),
                                                          C.c_void_p(out.ctypes.data)))
        return out

    def tree(self, task=0, replica=0) -> np.ndarray:
        """The whole sum-tree of one (replica, task) sub-ring: [2P] fp32 in heap order (node 1 = root, leaf i = node P + i)."""
        cap_t = self.capacity // max(self.core.cfg.num_tasks, 1)
        P = 1
        while P < cap_t:
            P *= 2
        out = np.empty(2 * P, dtype=np.float32)
        _lib.check(self.lib.b200sac_replay_get_tree(self._h, int(replica), int(task), out.size, C.c_void_p(out.ctypes.data)))
        return out

    def sample_prioritized(self, replica=0):
        """(s, a, r, s2, d, idx, w): one draw of the device PER sampler (its own draw counter), as CPU tensors."""
        c = self.core.cfg
        B = c.batch
        s, a, r = torch.empty(B, c.obs_dim), torch.empty(B, c.act_dim), torch.empty(B, 1)
        s2, d = torch.empty(B, c.obs_dim), torch.empty(B, 1)
        idx, w = torch.empty(B, dtype=torch.int64), torch.empty(B)
        _lib.check(self.lib.b200sac_replay_sample_prioritized(self._h, int(replica), _ptr(s), _ptr(a), _ptr(r), _ptr(s2), _ptr(d),
                                                              _ptr(idx), _ptr(w)))
        return s, a, r, s2, d, idx, w

    def refresh_priorities(self, seed, idx=None, replica=None, stochastic=True):
        """Recompute priorities with the current networks (b200sac_replay_refresh_priorities): the filled slots `idx` of one
        replica, or with idx=None every filled slot of every task; replica=None means every replica and needs idx=None (slot
        lists are per replica).  stochastic=False evaluates the TD target at the policy's mean action; True draws the next
        action's noise keyed by (seed, replica, slot).  Synchronous; sees every reset and recycle enqueued before it."""
        if idx is not None and replica is None:
            raise ValueError("refresh_priorities with idx= needs replica= (slot lists are per replica)")
        if not isinstance(stochastic, (bool, np.bool_)):
            raise ValueError(f"stochastic must be a bool, got {stochastic!r}")
        if idx is not None:
            idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1))
        for r in _replicas(self.core.cfg.replicas, replica):
            n, p = (0, C.c_void_p(0)) if idx is None else (idx.size, C.c_void_p(idx.ctypes.data))
            if idx is not None and n == 0:
                continue
            _lib.check(self.lib.b200sac_replay_refresh_priorities(self._h, int(r), n, p, C.c_uint64(int(seed) % (1 << 64)),
                                                                  1 if stochastic else 0, _stream()))

    # ---- prior-data rings (symmetric sampling) -------------------------------------------------
    def attach_prior(self, prior: Optional["Replay"]):
        """Make `prior` (a uniform, unlinked device Replay of the same core) this ring's prior-data ring, or detach with
        None.  Steps then take set_prior_rows(m) rows of every task block from the prior (0 until set).  The ring keeps a
        reference to the prior while it is attached."""
        if prior is not None and not isinstance(prior, Replay):
            raise ValueError(f"attach_prior takes a Replay or None (got {type(prior).__name__})")
        _lib.check(self.lib.b200sac_replay_attach_prior(self._h, None if prior is None else prior._h))
        self._prior = prior

    def set_prior_rows(self, m: int, replica=None):
        """Prior rows m in [0, batch / num_tasks] of every task block of one replica's steps (None: all), in stream order."""
        if isinstance(m, bool) or int(m) != m:
            raise ValueError(f"prior rows must be an int (got {m!r})")
        for r in _replicas(self.core.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_replay_set_prior_rows(self._h, r, int(m), _stream()))

    def get_prior_rows(self, replica=0) -> int:
        m = C.c_int32(0)
        _lib.check(self.lib.b200sac_replay_get_prior_rows(self._h, int(replica), C.byref(m)))
        return m.value

    # ---- n-step returns (ring with trajectory links) ---------------------------------------------
    def set_nstep(self, n: int, replica=None):
        """Horizon n in [1, 16] of one replica (None: all), in stream order: steps enqueued afterwards fold n-step returns."""
        for r in _replicas(self.core.cfg.replicas, replica):
            _lib.check(self.lib.b200sac_replay_set_nstep(self._h, r, int(n), _stream()))

    def get_nstep(self, replica=0) -> int:
        n = C.c_int32(0)
        _lib.check(self.lib.b200sac_replay_get_nstep(self._h, int(replica), C.byref(n)))
        return n.value

    def close_streams(self, streams, replica=0):
        """Forget the open tails of these stream ids: their next rows start new trajectories (for recycling ids)."""
        ids = np.ascontiguousarray(np.asarray(streams, dtype=np.int32).reshape(-1))
        if ids.size:
            _lib.check(self.lib.b200sac_replay_close_streams(self._h, int(replica), ids.size, C.c_void_p(ids.ctypes.data)))

    def links(self, task=0, replica=0) -> np.ndarray:
        """link[slot] of one (replica, task) sub-ring: the sub-ring-local slot of the successor transition, or -1."""
        out = np.empty(self.capacity // max(self.core.cfg.num_tasks, 1), dtype=np.int32)
        _lib.check(self.lib.b200sac_replay_get_links(self._h, int(replica), int(task), out.size, C.c_void_p(out.ctypes.data)))
        return out

    def fold(self, idx, replica=0):
        """(s, a, R, s2, d, disc, m) of ring slots `idx` as numpy arrays: the device's n-step fold with the replica's current
        horizon and gamma (the current stream is synchronised first, so a set_hparams enqueued on it has landed)."""
        torch.cuda.current_stream().synchronize()
        idx = np.ascontiguousarray(np.asarray(idx, dtype=np.int64).reshape(-1))
        c, n = self.core.cfg, idx.size
        s, a, R = np.empty((n, c.obs_dim), np.float32), np.empty((n, c.act_dim), np.float32), np.empty(n, np.float32)
        s2, d, disc = np.empty((n, c.obs_dim), np.float32), np.empty(n, np.float32), np.empty(n, np.float32)
        m = np.empty(n, np.int32)
        _lib.check(self.lib.b200sac_replay_fold(self._h, int(replica), n, *[C.c_void_p(t.ctypes.data) for t in
                                                                            (idx, s, a, R, s2, d, disc, m)]))
        return s, a, R, s2, d, disc, m
