"""Canonical parameter names <-> the reference's state_dict keys (the wire format).

`Player.pull_parameters` does `actor.load_state_dict(parameters['actor'])`
(/root/reference/LunarLander_Distributed_SAC/src/player.py:75-85) and
checkpoints store per-module state_dicts (.../learner.py:144-163), so the
reference's key names are a compatibility contract:

  LL / VS   Actor : layer_intermediate.{i}.weight|bias, mu_log_std_layer.weight|bias
                    (LunarLander_Distributed_SAC/src/model.py:20-24)
            Critic: first_layer.*, layer_module.{j}.*        (model.py:102-106)
  MS        Actor : mu_log_std_layer.{2i}.*                  (MT10_Distributed_MTSAC/src/model.py:27-33, utils.py:36-57)
            Critic: Q_function_1.{2i}.*, Q_function_2.{2i}.* (model.py:136-149)

Layer-normalized critics (critic_layer_norm) add a LayerNorm after every hidden Linear: `layer_norms.{i}.*` beside the LL / VS
Critic's Linear keys, and the natural nn.Sequential(Linear, LayerNorm, ReLU, ...) numbering Q_function_{w}.{3i}.* (Linear i),
Q_function_{w}.{3i+1}.* (its LayerNorm) for MS.  Dropout Q-functions (critic_dropout) keep the LL / VS keys (the dropout
has no parameters) and number MS as nn.Sequential(Linear, Dropout, LayerNorm, ReLU, ...): Q_function_{w}.{4i}.* (Linear i),
Q_function_{w}.{4i+2}.* (its LayerNorm).

Canonical names (used by the C ABI's layout table): `<net>.<i>.weight|bias`
with net in {actor,q1,q2,q1_target,q2_target}, `<net>.<i>.ln.weight|bias` for a critic's LayerNorm and `log_alpha`.
"""


def actor_key_map(family: str, n_layers: int):
    """{reference key: canonical key} for the actor; n_layers counts the head."""
    m = {}
    for i in range(n_layers):
        for kind in ("weight", "bias"):
            if family in ("LL", "VS"):
                ref = f"mu_log_std_layer.{kind}" if i == n_layers - 1 else f"layer_intermediate.{i}.{kind}"
            elif family == "MS":
                ref = f"mu_log_std_layer.{2 * i}.{kind}"
            else:
                raise ValueError(family)
            m[ref] = f"actor.{i}.{kind}"
    return m


def critic_key_map(family: str, n_layers: int, which: int, target: bool = False, layer_norm: bool = False,
                   dropout: bool = False):
    """{reference key: canonical key} for Q-function `which` (1|2; 1 .. E on a critic ensemble), in the canonical layout
    order; n_layers counts the head.

    LL/VS: keys of ONE Critic module (local_critic_{which});
    MS   : keys of the twin Critic module restricted to Q_function_{which}.
    layer_norm: the critics with a LayerNorm after every hidden Linear; dropout (with layer_norm): a Dropout between them
    (the module docstring gives the keys)."""
    if dropout and not layer_norm:
        raise ValueError("dropout=True describes the DroQ critics, which have layer_norm=True")
    if family not in ("LL", "VS", "MS"):
        raise ValueError(family)
    net = f"q{which}" + ("_target" if target else "")
    step = 4 if dropout else (3 if layer_norm else 2)      # MS: modules per hidden layer of the nn.Sequential
    m = {}
    for i in range(n_layers):
        for kind in ("weight", "bias"):
            if family in ("LL", "VS"):
                ref = f"first_layer.{kind}" if i == 0 else f"layer_module.{i - 1}.{kind}"
            else:
                ref = f"Q_function_{which}.{step * i}.{kind}"
            m[ref] = f"{net}.{i}.{kind}"
        if layer_norm and i < n_layers - 1:
            for kind in ("weight", "bias"):
                ref = f"layer_norms.{i}.{kind}" if family in ("LL", "VS") else f"Q_function_{which}.{step * i + step - 2}.{kind}"
                m[ref] = f"{net}.{i}.ln.{kind}"
    return m


def care_encoder_key_map(n_mix: int, n_trunk: int, n_ctx: int, prefix: str):
    """{reference key under `state_encoder.`: canonical key} for one CARE state encoder
    (MT10_Distributed_CARE/src/state_encoder.py:36-63,196-217: mixtureEncoders.{2l}.{W,b}, trunk.{2j}.*, mlp_context.{2j}.*).
    prefix = 'cse' (critic's; also what the actor's tied copy exports) or 'tse' (target critic's)."""
    m = {}
    for l in range(n_mix):
        m[f"state_encoder.mixture_encoders.mixtureEncoders.{2 * l}.W"] = f"{prefix}.mix.{l}.W"
        m[f"state_encoder.mixture_encoders.mixtureEncoders.{2 * l}.b"] = f"{prefix}.mix.{l}.b"
    for name, n, ref in (("trunk", n_trunk, "trunk"), ("ctx", n_ctx, "mlp_context")):
        for j in range(n):
            for kind in ("weight", "bias"):
                m[f"state_encoder.{ref}.{2 * j}.{kind}"] = f"{prefix}.{name}.{j}.{kind}"
    return m
