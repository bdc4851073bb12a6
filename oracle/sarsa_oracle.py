"""oracle/sarsa_oracle.py — CPU restatement of DeepSARSA and of SARSAReplayBuffer's delayed push
(TEST INFRASTRUCTURE ONLY; eager PyTorch fp32 like the reference).

Restated reference sites (paths relative to the Pearl source tree):
  policy_learners/sequential_decision_making/deep_sarsa.py:58-75           next-state values Q_target(s', one_hot(a'))
  policy_learners/sequential_decision_making/deep_td_learning.py:269-360   forward (target update first), loss, learn_batch
  policy_learners/policy_learner.py:162-215                                learn loop, batch clamp, preprocess_batch
  replay_buffers/sequential_decision_making/sarsa_replay_buffer.py:29-101  the delayed-push state machine
  replay_buffers/tensor_based_replay_buffer.py:253-288                     sample, clear (the cache survives it)
  pearl_agent.py:213-220                                                   on-policy learners clear the buffer after learn()
Per round: when (training_steps + 1) % target_update_freq == 0 the soft target update with the CURRENT online parameters;
q = Q(s, a); y = Q'(s', a') gamma (1 - terminated) + r with a' the committed next action (no max, no available sets);
loss = MSE(q, y); one AdamW(amsgrad) step; reported loss mean |q - y|.  Parity with the reference is pinned by
tests/golden/sarsa_*.npz (oracle/gen_sarsa_golden.py).
"""
from __future__ import annotations

import random
from collections import deque

import torch
import torch.nn.functional as F

from .pearl_oracle import OracleDQN, flat, load_flat  # noqa: F401


class OracleSARSABuffer:
    """SARSAReplayBuffer: FIFO deque of complete SARSA tuples behind a one-entry cache, sampled with random.sample."""

    def __init__(self, capacity: int) -> None:
        self.capacity = capacity
        self.memory: deque = deque([], maxlen=capacity)
        self.cache = None

    def __len__(self) -> int:
        return len(self.memory)

    def clear(self) -> None:                       # the cache is kept
        self.memory = deque([], maxlen=self.capacity)

    def push(self, state, action, reward, terminated, truncated, next_state) -> list:
        """One push; returns the tuples it appended (state, action, reward, next_state, next_action, terminated, truncated)."""
        state = torch.as_tensor(state, dtype=torch.float32).reshape(-1).clone()
        next_state = torch.as_tensor(next_state, dtype=torch.float32).reshape(-1).clone()
        row = (state, int(action), float(reward), next_state, None, bool(terminated), bool(truncated))
        out = []
        if self.cache is not None and torch.equal(self.cache[3], state):
            out.append(self.cache[:4] + (int(action),) + self.cache[5:])
        if not (terminated or truncated):
            self.cache = row
        else:
            out.append(row[:4] + (int(action),) + row[5:])
        self.memory.extend(out)
        return out

    def sample(self, batch_size: int) -> dict:
        if batch_size > len(self):
            raise ValueError(f"Can't get a batch of size {batch_size} from a replay buffer with only {len(self)} elements")
        cols = list(zip(*random.sample(self.memory, batch_size)))
        return dict(state=torch.stack(cols[0]), action=torch.tensor(cols[1]), reward=torch.tensor(cols[2], dtype=torch.float32),
                    next_state=torch.stack(cols[3]), next_action=torch.tensor(cols[4]), terminated=torch.tensor(cols[5]),
                    truncated=torch.tensor(cols[6]))


class OracleSARSA(OracleDQN):
    """DeepSARSA.  `learn_batch(b)` takes the batch as preprocess_batch leaves it: state [B, O], action and next_action
    one-hot [B, A], reward [B], next_state [B, O], terminated [B] bool; the update schedule reads `self.training_steps`."""

    def _next_values(self, b):
        with torch.no_grad():
            return self._q_values(self.Qt, b["next_state"], b["next_action"])

    def learn(self, buf: OracleSARSABuffer, on_policy_clear: bool = True) -> dict:
        """PearlAgent.learn: PolicyLearner.learn, then clear() (DeepSARSA is on-policy)."""
        if len(buf) == 0:
            return {}
        bs = len(buf) if (self.batch_size == -1 or len(buf) < self.batch_size) else self.batch_size
        report = {"loss": []}
        for _ in range(self.training_rounds):
            self.training_steps += 1
            report["loss"].append(self.learn_batch(one_hot(buf.sample(bs), self.A)))
        if on_policy_clear:
            buf.clear()
        return report


def one_hot(b: dict, A: int) -> dict:
    """preprocess_batch: action and next_action through the one-hot representation."""
    oh = lambda x: F.one_hot(torch.as_tensor(x).long().reshape(-1), A).float()  # noqa: E731
    return dict(b, action=oh(b["action"]), next_action=oh(b["next_action"]))
