"""Developer tool: rates of the LinearBandit learner (pearl_b200.B200LinearBandit over a B200ReplayBuffer) on one GPU, next
to the eager-torch restatement (oracle/bandit_oracle.py) on the host:
  cb_step     the CB benchmark's loop (obs 16, 26 actions as a 5-bit binary code, batch 128, training_rounds 10, UCB
              alpha 1): time per environment step (act + push + learn()), and rounds/s of learn() alone
  scores      get_scores latency for 1 state and for 4096 states x 26 actions
  stress      obs 119, 8 actions one-hot (d = 128), batch 256: rounds/s of learn()
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after warm-up.  Prints the
card's name and power limit with the numbers.

    python tools/bandit_bench.py [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import torch  # noqa: E402

import pearl_b200 as P  # noqa: E402
from oracle import bandit_oracle as bo  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def timed(fn, min_s=2.0):
    """(calls, seconds) of fn() repeated until CUDA events span at least min_s."""
    fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    n = 1
    while True:
        e0.record()
        for _ in range(n):
            fn()
        e1.record()
        e1.synchronize()
        s = e0.elapsed_time(e1) / 1e3
        if s >= min_s:
            return n, s
        n = max(n * 2, int(n * min_s / max(s, 1e-6)) + 1)


class Space:
    def __init__(self, n):
        self.n = n
        self.actions = [torch.tensor([i]) for i in range(n)]
        self.actions_batch = torch.arange(n).view(n, 1)


def learner(obs, A, rep, B, rounds):
    mod = P.OneHotActionTensorRepresentationModule(A) if rep == "one_hot" else P.BinaryActionTensorRepresentationModule(rep)
    return P.B200LinearBandit(feature_dim=obs + mod.representation_dim, exploration_module=P.UCBExploration(1.0),
                              training_rounds=rounds, batch_size=B, action_representation_module=mod).to("cuda:0")


def filled(obs, A, n):
    g = torch.Generator().manual_seed(0)
    buf = P.B200ReplayBuffer(max(n, 1), rng="device")
    buf.push_batch(torch.randn(n, obs, generator=g), torch.randint(0, A, (n,), generator=g), torch.randn(n, generator=g), None,
                   torch.ones(n, dtype=torch.bool), torch.zeros(n, dtype=torch.bool), max_number_actions=A)
    buf.seed(0)
    return buf


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    res = {"card": card()}
    # cb_step: act + push + learn() per environment step
    lb, buf, sp = learner(16, 26, 5, 128, 10), filled(16, 26, 2048), Space(26)
    st = torch.randn(16, device="cuda:0")

    def step():
        a = int(lb.act(st, sp).reshape(-1)[0])
        buf.push(st, a, 1.0, True, False, max_number_actions=26)
        lb.learn(buf)
    n, s = timed(step)
    res["cb_step_us"] = 1e6 * s / n
    n, s = timed(lambda: lb.learn(buf))
    res["cb_learn_rounds_per_s"] = 10 * n / s
    # scores
    for m in (1, 4096):
        states = torch.randn(m, 16, device="cuda:0")
        n, s = timed(lambda: lb.get_scores(states, sp))
        res[f"scores_{m}x26_us"] = 1e6 * s / n
    # stress
    lb2, buf2 = learner(119, 8, "one_hot", 256, 100), filled(119, 8, 8192)
    n, s = timed(lambda: lb2.learn(buf2))
    res["stress_learn_rounds_per_s"] = 100 * n / s
    # the eager restatement on the host, one round at each shape
    for name, (k, B) in {"cb": (21, 128), "stress": (127, 256)}.items():
        o, x, y = bo.Ridge(k + 1, 1.0), torch.randn(B, k), torch.randn(B)
        t0, reps = time.perf_counter(), 0
        while time.perf_counter() - t0 < 2.0:
            o.round(x, y)
            reps += 1
        res[f"host_eager_{name}_rounds_per_s"] = reps / (time.perf_counter() - t0)
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "bandit_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
