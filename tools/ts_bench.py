"""Developer tool: Thompson sampling on the ridge learners against UCB on the same learners, on one GPU:
  neural_ts / neural_ucb   the CB benchmark's NeuralTS and NeuralLinUCB configs (obs 16, 26 actions as a 5-bit binary
                           code, hidden [64, 16], lr 0.01, batch 128, training_rounds 10; ThompsonSamplingExplorationLinear
                           with its defaults, UCBExploration alpha 1)
  lin_ts / lin_ts_eff / lin_ucb   LinearBandit (LinTS with default and efficient sampling, LinUCB) on the same rows,
                           training_rounds 10, batch 128
For each: the time of one environment step (act + push + learn()) and of one act for a single state.  A Thompson call
reads one status word back from the device; `status_readback_us` is that 4-byte copy alone on an idle stream (host
clock).  Times come from CUDA events around whole calls, over windows of at least 2 s after warm-up.  Prints the card's
name, power limit and maximum SM clock with the numbers.

    python tools/ts_bench.py [--out DIR]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import pearl_b200 as P  # noqa: E402
from tools.bandit_bench import Space, card, filled, timed  # noqa: E402


def learners():
    mod = lambda: P.BinaryActionTensorRepresentationModule(5)  # noqa: E731
    nl = lambda ex: P.B200NeuralLinearBandit(feature_dim=16 + 5, hidden_dims=[64, 16], learning_rate=0.01, batch_size=128,  # noqa: E731
                                             training_rounds=10, state_features_only=False, exploration_module=ex,
                                             action_representation_module=mod()).to("cuda:0")
    lin = lambda ex: P.B200LinearBandit(feature_dim=16 + 5, training_rounds=10, batch_size=128, exploration_module=ex,  # noqa: E731
                                        action_representation_module=mod()).to("cuda:0")
    return {"neural_ts": nl(P.ThompsonSamplingExplorationLinear()), "neural_ucb": nl(P.UCBExploration(1.0)),
            "lin_ts": lin(P.ThompsonSamplingExplorationLinear()),
            "lin_ts_eff": lin(P.ThompsonSamplingExplorationLinear(enable_efficient_sampling=True)),
            "lin_ucb": lin(P.UCBExploration(1.0))}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    res = {"card": card()}
    sp = Space(26)
    st = torch.randn(16, device="cuda:0")
    for name, pl in learners().items():
        buf = filled(16, 26, 2048)

        def step():
            a = int(pl.act(st, sp).reshape(-1)[0])
            buf.push(st, a, 1.0, True, False, max_number_actions=26)
            pl.learn(buf)
        n, s = timed(step)
        res[f"{name}_step_us"] = 1e6 * s / n
        n, s = timed(lambda: pl.act(st, sp))
        res[f"{name}_act_us"] = 1e6 * s / n
    status = torch.zeros(1, dtype=torch.int32, device="cuda:0")
    torch.cuda.synchronize()
    t0, reps = time.perf_counter(), 0
    while time.perf_counter() - t0 < 2.0:
        status.item()
        reps += 1
    res["status_readback_us"] = 1e6 * (time.perf_counter() - t0) / reps
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "ts_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
