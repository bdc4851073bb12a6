"""The conservative (CQL) path of B200DeepQLearning / B200DoubleDQN: Pearl's DeepQLearning / DoubleDQN built with
`is_conservative=True, conservative_alpha=alpha` (policy_learners/sequential_decision_making/deep_td_learning.py:269-360
with utils/functional_utils/learning/loss_fn_utils.py:17-71), on an H100 through `prl_cql_*` (csrc/cql.cu).

The DQN plugin (dqn.py) keeps its binding: `_Q`, `_Q_target` and the AdamW state are views into the flat vectors it
allocates, and a checkpoint or lr change is picked up the same way.  When `_is_conservative` is set, the plugin hands the
flat vectors to a `prl_cql` handle instead of a `prl_dqn` one: `learn` (over a B200ReplayBuffer) and `q_values` run
through its prl_cql_* entry points, `learn_batch` is the function here.  A round updates the target first (in the rounds
the reference's schedule flags), then takes one AdamW(amsgrad) step on mean (q - y)^2 + alpha * cql, with the reference's
CQL term as it computes it (include/pearl_b200.h).  alpha is read from `_conservative_alpha` on every call.  No CPU
fallback."""
from __future__ import annotations

from . import _lib
from ._batch import check_features, dense_rows, next_available_first, plugin_call, slot_ids

PREFIX = "prl_cql_"
NAME = "conservative (CQL) DQN"
LAUNCH_INFO = dict(launches="last_launches")


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the conservative configurations the CUDA learner does not run or the reference rejects."""
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no conservative (CQL) kernel: use engine='auto' or 'simt'")
    alpha(pl)
    if pl._n_actions < 2:
        raise ValueError("conservative (CQL) updates need at least 2 actions: the reference's CQL term gathers column 1 "
                         "of the current-action values")


def alpha(pl) -> float:
    a = getattr(pl, "_conservative_alpha", None)
    if a is None:
        raise ValueError("conservative_alpha is None: the reference's CQL loss multiplies it with the CQL term")
    return float(a)


def learn_args(pl) -> tuple:
    """The arguments prl_cql_learn takes after the training-step count: alpha."""
    return (alpha(pl),)


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.CqlCfg:
    return _lib.CqlCfg(obs_dim=pl._obs_dim, n_actions=pl._n_actions, hidden1=pl._hidden[0], hidden2=pl._hidden[1],
                       double_dqn=int(pl._double), target_update_freq=int(pl._target_update_freq), max_batch=max_batch,
                       max_rounds=pl._max_rounds, lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"],
                       weight_decay=hp["weight_decay"], gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` with the CQL term on a caller-supplied batch (raw ids, or the one-hot tensors the
    reference's preprocess_batch produces).  `curr_available_actions` (padding included: the reference's CQL term ignores
    `curr_unavailable_actions_mask`) defaults to every action; next-action slots that are masked are compacted away in
    order, which keeps DoubleDQN's first argmax."""
    B, A = len(batch), pl._n_actions
    check_features(batch, pl._obs_dim)
    pl._bind(B)
    dev = pl._device
    cur = slot_ids(batch, "curr_available_actions", B, A, dev)
    return plugin_call(pl, B, *dense_rows(batch, B, A, dev), cur, *next_available_first(batch, B, A, dev),
                       int(pl._training_steps), alpha(pl))
