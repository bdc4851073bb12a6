"""Developer tool: rates of the NeuralLinearBandit learner (pearl_b200.B200NeuralLinearBandit over a B200ReplayBuffer) on
one GPU, next to the eager-torch restatement (oracle/neural_linear_oracle.py) on the host:
  cb_step     the CB benchmark's config (obs 16, 26 actions as a 5-bit binary code, hidden [64, 16], lr 0.01, batch 128,
              training_rounds 10, UCB alpha 1, state_features_only=False): time per environment step (act + push +
              learn()), and rounds/s of learn() alone
  scores      get_scores latency for 1 state and for 4096 states x 26 actions
  wide        input 127 (state alone), hidden [256, 127], batch 256: rounds/s of learn()
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after warm-up.  Prints the
card's name, power limit and maximum SM clock with the numbers.

    python tools/neural_linear_bench.py [--out DIR]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import pearl_b200 as P  # noqa: E402
from oracle import neural_linear_oracle as no  # noqa: E402
from tools.bandit_bench import Space, card, filled, timed  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    # cb_step: act + push + learn() per environment step, the CB benchmark's config
    mod = P.BinaryActionTensorRepresentationModule(5)
    nl = P.B200NeuralLinearBandit(feature_dim=16 + 5, hidden_dims=[64, 16], learning_rate=0.01, batch_size=128, training_rounds=10,
                                  state_features_only=False, exploration_module=P.UCBExploration(1.0),
                                  action_representation_module=mod).to("cuda:0")
    buf, sp = filled(16, 26, 2048), Space(26)
    st = torch.randn(16, device="cuda:0")

    def step():
        a = int(nl.act(st, sp).reshape(-1)[0])
        buf.push(st, a, 1.0, True, False, max_number_actions=26)
        nl.learn(buf)
    n, s = timed(step)
    res["cb_step_us"] = 1e6 * s / n
    n, s = timed(lambda: nl.learn(buf))
    res["cb_learn_rounds_per_s"] = 10 * n / s
    for m in (1, 4096):
        states = torch.randn(m, 16, device="cuda:0")
        n, s = timed(lambda: nl.get_scores(states, sp))
        res[f"scores_{m}x26_us"] = 1e6 * s / n
    # wide: the state alone, input 127, hidden [256, 127], batch 256
    wide = P.B200NeuralLinearBandit(feature_dim=127, hidden_dims=[256, 127], batch_size=256, training_rounds=100).to("cuda:0")
    buf2 = filled(127, 8, 8192)
    n, s = timed(lambda: wide.learn(buf2))
    res["wide_learn_rounds_per_s"] = 100 * n / s
    # the eager restatement on the host, one round at each shape
    for name, (f, h1, h2, B) in {"cb": (21, 64, 16, 128), "wide": (127, 256, 127, 256)}.items():
        n_par = sum(int(torch.tensor(x).prod()) for x in no.shapes(f, h1, h2))
        o = no.NeuralLinear(torch.randn(n_par) * 0.1, f, h1, h2, lr=0.01)
        x, y = torch.randn(B, f), torch.randn(B)
        t0, reps = time.perf_counter(), 0
        while time.perf_counter() - t0 < 2.0:
            o.round(x, y)
            reps += 1
        res[f"host_eager_{name}_rounds_per_s"] = reps / (time.perf_counter() - t0)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "neural_linear_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
