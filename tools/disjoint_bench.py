"""Developer tool: the disjoint linear bandits on one GPU, against the eager-torch reference on the host.
  dlb_agent        test_agent.py's DisjointLinearBandit (obs 3, 3 actions tensor([i]), feature_dim 4, DisjointUCBExploration
                   alpha 0.1, batch 1, training_rounds 1) as an act -> push -> learn() loop: time per environment step
  container26      a DisjointBanditContainer of 26 LinearBandit arms, obs 16, batch 128, training_rounds 10 (the CB
                   benchmark's obs and action count): time per learn() and per act of one state
  arms128          128 LinearBandit arms at feature_dim 127 (d = 128), batch 4096: learn() rounds per second, next to one
                   B200LinearBandit round at d = 128 on 4096 rows (learn_batch) in the same run; and the round alone
                   (prl_dcb_learn_batch with no report, graph replay) for 128 arms and for 1 arm at the same shape
  *_host_ms        oracle/disjoint_oracle.py's eager-torch restatement of one round (the reference's per-arm loop) on the
                   host CPU, for the same shapes
Times come from CUDA events around whole calls (host clock for the CPU rows), over windows of at least 2 s after
warm-up.  Prints the card's name, power limit, current and maximum SM clock with the numbers.

    python tools/disjoint_bench.py [--out DIR]
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
from oracle import disjoint_oracle as do  # noqa: E402
from tools.bandit_bench import Space, filled, timed  # noqa: E402


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def host_ms(fn, min_s=2.0):
    fn()
    n, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < min_s:
        fn()
        n += 1
    return 1e3 * (time.perf_counter() - t0) / n


def container(K, obs, B, rounds):
    arms = [P.B200LinearBandit(feature_dim=obs) for _ in range(K)]
    return P.B200DisjointBanditContainer(feature_dim=obs, arm_bandits=arms, exploration_module=P.DisjointUCBExploration(1.0),
                                         training_rounds=rounds, batch_size=B)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    torch.cuda.set_device(0)
    torch.manual_seed(0)
    res = {"card": card()}
    g = torch.Generator().manual_seed(0)

    # test_agent's DisjointLinearBandit loop
    lb = P.B200DisjointLinearBandit(feature_dim=4, action_space=Space(3), exploration_module=P.DisjointUCBExploration(0.1),
                                    batch_size=1, training_rounds=1)
    buf = filled(3, 3, 1024)
    st = torch.randn(3, device="cuda:0")

    def step():
        a = int(lb.act(st, Space(3)).reshape(-1)[0])
        buf.push(st, a, 1.0, True, False, max_number_actions=3)
        lb.learn(buf)
    n, s = timed(step)
    res["dlb_agent_step_us"] = 1e6 * s / n
    ref = do.Disjoint(3, 5, [1.0] * 3, linear=True)
    x1, a1, r1 = torch.randn(1, 3), torch.tensor([[1]]), torch.randn(1)
    feat = torch.arange(3, dtype=torch.float32).reshape(3, 1)
    res["dlb_agent_learn_host_ms"] = host_ms(lambda: ref.round(x1, a1, r1, None, feat))

    # 26 arms, obs 16, batch 128, 10 rounds
    dc = container(26, 16, 128, 10)
    buf = filled(16, 26, 2048)
    n, s = timed(lambda: dc.learn(buf))
    res["container26_learn_ms"] = 1e3 * s / n
    st = torch.randn(16, device="cuda:0")
    n, s = timed(lambda: dc.act(st, Space(26)))
    res["container26_act_us"] = 1e6 * s / n
    ref = do.Disjoint(26, 17, [1.0] * 26)
    X, A, R = torch.randn(128, 16, generator=g), torch.randint(0, 26, (128, 1), generator=g), torch.randn(128, generator=g)
    res["container26_round_host_ms"] = host_ms(lambda: ref.round(X, A, R))

    # 128 arms at d = 128, batch 4096, against one LinearBandit round at d = 128
    dc = container(128, 127, 4096, 10)
    buf = filled(127, 128, 16384)
    n, s = timed(lambda: dc.learn(buf))
    res["arms128_d128_b4096_rounds_per_s"] = 10 * n / s
    # the round alone: prl_dcb_learn_batch on a dense batch with no report (one round's launches, no host work beyond
    # the launch), against the same call for a one-arm learner of the same width
    from pearl_b200 import _lib
    from pearl_b200.replay_buffer import _stream_ptr

    def round_only(K):
        c = container(K, 127, 4096, 1)
        xs, rw = torch.randn(4096, 127, device="cuda:0"), torch.randn(4096, device="cuda:0")
        ids = torch.randint(0, K, (4096,), device="cuda:0", dtype=torch.int32)
        c.learn_batch(P.TransitionBatch(state=xs, action=ids.long().reshape(-1, 1), reward=rw))
        rg, p, st = c._dj, _lib.ptr, _stream_ptr(torch.device("cuda:0"))
        return timed(lambda: _lib.check(rg.lib.prl_dcb_learn_batch(rg.handle, 4096, p(xs), 0, p(ids), p(rw), None, None,
                                                                    None, None, None, st)))
    n, s = round_only(128)
    res["arms128_d128_b4096_round_only_us"] = 1e6 * s / n
    n, s = round_only(1)
    res["arms1_d128_b4096_round_only_us"] = 1e6 * s / n
    one = P.B200LinearBandit(feature_dim=127, batch_size=4096).to("cuda:0")
    batch = P.TransitionBatch(state=torch.randn(4096, 127, device="cuda:0"), action=torch.zeros(4096, 0, device="cuda:0"),
                              reward=torch.randn(4096, 1, device="cuda:0"))
    n, s = timed(lambda: one.learn_batch(batch))
    res["linear_d128_b4096_rounds_per_s"] = n / s
    ref = do.Disjoint(128, 128, [1.0] * 128)
    X, A, R = torch.randn(4096, 127, generator=g), torch.randint(0, 128, (4096, 1), generator=g), torch.randn(4096, generator=g)
    res["arms128_round_host_ms"] = host_ms(lambda: ref.round(X, A, R))

    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "disjoint_bench.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
