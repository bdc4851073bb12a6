"""The DeepSARSA path of the DQN plugin: Pearl's DeepSARSA (policy_learners/sequential_decision_making/deep_sarsa.py on
deep_td_learning.py:269-360), on an H100 through `prl_sarsa_*` (csrc/sarsa.cu).

B200DeepSARSA (dqn.py) keeps the DQN plugin's binding: `_Q`, `_Q_target` and the AdamW state are views into the flat
vectors it allocates, and a checkpoint or lr change is picked up the same way; the flat vectors go to a `prl_sarsa`
handle.  `learn` runs over a B200SARSAReplayBuffer (the ring stores the committed next action), `learn_batch` is the
function here.  A round updates the target first (in the rounds the reference's schedule flags), then takes one
AdamW(amsgrad) step on mean (q - y)^2 with y = r + gamma (1 - terminated) Q'(s', a').  No CPU fallback."""
from __future__ import annotations

from . import _lib
from ._batch import check_features, dense_rows, plugin_call, staged_ids

PREFIX = "prl_sarsa_"
NAME = "DeepSARSA"
LAUNCH_INFO = dict(launches="last_launches", graph_captures="graph_captures")


def check_config(pl, engine: str) -> None:
    """Refuses, at construction, the configurations the SARSA learner does not run."""
    if engine == "tc":
        raise NotImplementedError("engine='tc' has no DeepSARSA kernel: use engine='auto' or 'simt'")
    if getattr(pl, "_is_conservative", False):
        raise NotImplementedError("DeepSARSA with is_conservative=True (CQL) is not supported")
    if pl._dueling:
        raise NotImplementedError("DeepSARSA with a DuelingQValueNetwork is not supported")
    if getattr(pl, "_multihead", False):
        raise NotImplementedError("DeepSARSA with a VanillaQValueMultiHeadNetwork is not supported")


def make_cfg(pl, hp: dict, max_batch: int) -> _lib.SarsaCfg:
    return _lib.SarsaCfg(obs_dim=pl._obs_dim, n_actions=pl._n_actions, hidden1=pl._hidden[0], hidden2=pl._hidden[1],
                         target_update_freq=int(pl._target_update_freq), max_batch=max_batch, max_rounds=pl._max_rounds,
                         lr=hp["lr"], beta1=hp["beta1"], beta2=hp["beta2"], eps=hp["eps"], weight_decay=hp["weight_decay"],
                         gamma=float(pl._discount_factor), tau=float(pl._soft_update_tau))


def learn_args(pl) -> tuple:
    return ()


def learn_batch(pl, batch) -> dict:
    """`DeepTDLearning.learn_batch` with DeepSARSA's next-state values on a caller-supplied batch (raw ids, or the one-hot
    tensors the reference's preprocess_batch produces).  `next_action` is required, as the reference asserts; the
    available action sets take no part."""
    if getattr(batch, "next_action", None) is None:
        raise AssertionError("SARSA needs to have next action")
    B, A = len(batch), pl._n_actions
    check_features(batch, pl._obs_dim)
    pl._bind(B)
    dev = pl._device
    state, action, reward, next_state, term = dense_rows(batch, B, A, dev)
    next_action = staged_ids(batch.next_action, A, (B,), dev, "batch.next_action")
    return plugin_call(pl, B, state, action, reward, next_state, next_action, term, int(pl._training_steps))
