"""Developer tool: rates of the NeuralBandit learner (pearl_b200.B200NeuralBandit over a B200ReplayBuffer) on one GPU, next
to the eager-torch restatement (oracle/neural_bandit_oracle.py) on the host:
  cb_step     the CB benchmark's SquareCB config (obs 16, 26 actions as a 5-bit binary code, hidden [64, 16], lr 0.01,
              batch 128, training_rounds 10, gamma = 10 sqrt(10000 x 21)): time per environment step (act + push +
              learn()), and rounds/s of learn() alone
  act         SquareCB act latency for one state
  scores      get_scores latency for 4096 states x 26 actions
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after warm-up.  Prints the
card's name, power limit and maximum SM clock with the numbers.

    python tools/neural_bandit_bench.py [--out DIR]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import pearl_b200 as P  # noqa: E402
from oracle import neural_bandit_oracle as no  # noqa: E402
from tools.bandit_bench import Space, card, filled, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    mod = P.BinaryActionTensorRepresentationModule(5)
    gamma = 10.0 * (10000 * 21) ** 0.5
    nb = P.B200NeuralBandit(feature_dim=16 + 5, hidden_dims=[64, 16], learning_rate=0.01, batch_size=128, training_rounds=10,
                            exploration_module=P.SquareCBExploration(gamma=gamma), action_representation_module=mod).to("cuda:0")
    buf, sp = filled(16, 26, 2048), Space(26)
    st = torch.randn(16, device="cuda:0")

    def step():
        a = int(nb.act(st, sp))
        buf.push(st, a, 1.0, True, False, max_number_actions=26)
        nb.learn(buf)
    n, s = timed(step)
    res["cb_step_us"] = 1e6 * s / n
    n, s = timed(lambda: nb.learn(buf))
    res["cb_learn_rounds_per_s"] = 10 * n / s
    n, s = timed(lambda: nb.act(st, sp))
    res["act_1_state_us"] = 1e6 * s / n
    states = torch.randn(4096, 16, device="cuda:0")
    n, s = timed(lambda: nb.get_scores(states, sp))
    res["scores_4096x26_us"] = 1e6 * s / n
    # the eager restatement on the host, one round at the benchmark's shape
    f, h1, h2, B = 21, 64, 16, 128
    n_par = sum(int(torch.tensor(x).prod()) for x in no.shapes(f, h1, h2))
    o = no.NeuralBandit(torch.randn(n_par) * 0.1, f, h1, h2, lr=0.01)
    x, y = torch.randn(B, f), torch.randn(B)
    t0, reps = time.perf_counter(), 0
    while time.perf_counter() - t0 < 2.0:
        o.round(x, y)
        reps += 1
    res["host_eager_cb_rounds_per_s"] = reps / (time.perf_counter() - t0)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "neural_bandit_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
