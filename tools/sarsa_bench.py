"""Developer tool: rates of the DeepSARSA learner (pearl_b200.B200DeepSARSA over a B200SARSAReplayBuffer) on one GPU,
next to the eager-torch restatement (oracle/sarsa_oracle.py) on the host:
  SARSA_method  the shape of Pearl's SARSA_method benchmark (obs 4, 2 actions, [64, 64], batch 32): gradient-steps/s of
                learn() over a filled buffer
  stress        obs 128, 16 actions, [256, 256], batch 256: gradient-steps/s of learn()
  on_policy     SARSA_method's shape the way PearlAgent runs it: per episode (lengths 5-60, so the batch follows the
                episode length below 32) push the episode, learn() with training_rounds 1, clear(); learn() calls/s
                (CUDA events around learn() alone), the graph captures of the run, and the cost of one capture (host
                clock around a learn() at a new batch size, minus a replay of a size seen before)
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up call.  Prints
the card's name and power limit with the numbers.

    python tools/sarsa_bench.py [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import numpy as np  # noqa: E402
import torch  # noqa: E402

import pearl_b200  # noqa: E402
from oracle.sarsa_oracle import OracleSARSA, one_hot  # noqa: E402

SHAPES = {"SARSA_method": dict(obs=4, A=2, hidden=64, B=32, n=100_000),
          "stress": dict(obs=128, A=16, hidden=256, B=256, n=200_000)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(shape, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    n, obs, A = shape["n"], shape["obs"], shape["A"]
    return dict(state=rng.standard_normal((n, obs), dtype=np.float32), next_state=rng.standard_normal((n, obs), dtype=np.float32),
                reward=rng.standard_normal(n, dtype=np.float32), term=rng.random(n) < 0.01, trunc=np.zeros(n, bool),
                action=rng.integers(0, A, size=n).astype(np.int32), next_action=rng.integers(0, A, size=n).astype(np.int32))


class Space:
    def __init__(self, A):
        self.n, self.actions, self.actions_batch = A, [torch.tensor([i]) for i in range(A)], torch.arange(A).view(A, 1)


def learner(shape, rounds):
    h, A = shape["hidden"], shape["A"]
    torch.manual_seed(3)
    return pearl_b200.B200DeepSARSA(state_dim=shape["obs"], action_space=Space(A), hidden_dims=[h, h], training_rounds=rounds,
                                    batch_size=shape["B"],
                                    action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(A)).to("cuda:0")


def push(buf, d, i, A):
    t = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
    buf.push_batch(t("state"), t("action"), t("reward"), t("next_state"), t("term"), t("trunc"), max_number_actions=A,
                   next_action=t("next_action"))


def timed(fn, per_call, window_s=2.0):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    done, ms = 0, 0.0
    while ms < window_s * 1e3:
        e0.record()
        fn()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        done += per_call
    return done / (ms / 1e3), ms / 1e3


def gpu_rate(shape, d, rounds_per_call=200):
    buf = pearl_b200.B200SARSAReplayBuffer(shape["n"], rng="device")
    push(buf, d, np.arange(shape["n"]), shape["A"])
    buf.seed(1)
    pl = learner(shape, rounds_per_call)
    rep = pl.learn(buf, trace=True)                             # warm-up: capture, module loads
    rate, win = timed(lambda: pl.learn(buf), rounds_per_call)
    return dict(steps_per_s=rate, window_s=win, launches_per_round=rep["launches"] / rounds_per_call)


def on_policy(shape, d, window_s=2.0):
    """PearlAgent's loop for an on-policy learner: push an episode, learn(), clear()."""
    A, rng = shape["A"], np.random.Generator(np.random.PCG64(11))
    pl = learner(shape, 1)
    buf = pearl_b200.B200SARSAReplayBuffer(1000, rng="device")
    lengths = rng.integers(5, 61, size=4096)
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    pos, k, ms, calls = 0, 0, 0.0, 0

    def episode():
        nonlocal pos, k
        L = int(lengths[k % len(lengths)])
        k += 1
        push(buf, d, np.arange(pos, pos + L) % shape["n"], A)
        pos += L
    episode()
    pl.learn(buf)                                               # warm-up call
    buf.clear()
    torch.cuda.synchronize()
    while ms < window_s * 1e3:
        episode()
        e0.record()
        pl.learn(buf)
        e1.record()
        e1.synchronize()
        buf.clear()
        ms += e0.elapsed_time(e1)
        calls += 1
    captures = pl.launch_info()["graph_captures"]
    # one capture: learn() at batch sizes the cache has not seen (a fresh learner with batch_size 64, sizes 33..40), minus
    # learn() at a size it has (a replay)
    pl2 = learner(dict(shape, B=64), 1)
    cost = []
    for L in range(33, 41):
        buf.clear()
        push(buf, d, np.arange(L), A)
        for rep in range(2):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            pl2.learn(buf)
            torch.cuda.synchronize()
            cost.append(time.perf_counter() - t0)
    first, replay = np.asarray(cost[0::2]), np.asarray(cost[1::2])
    return dict(learn_calls_per_s=calls / (ms / 1e3), window_s=ms / 1e3, episodes=calls + 1, graph_captures=captures,
                distinct_batch_sizes=len({min(int(L), shape["B"]) for L in lengths[:k]}),
                capture_ms=float(np.median(first - replay) * 1e3), replay_call_ms=float(np.median(replay) * 1e3))


def host_rate(shape, d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    h, A = shape["hidden"], shape["A"]
    orc = OracleSARSA(shape["obs"], A, (h, h))
    rng = np.random.Generator(np.random.PCG64(5))
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or steps < 3:
        i = rng.choice(shape["n"], size=shape["B"], replace=False)
        b = {k: torch.from_numpy(d[src][i]) for k, src in (("state", "state"), ("action", "action"), ("reward", "reward"),
                                                            ("next_state", "next_state"), ("next_action", "next_action"),
                                                            ("terminated", "term"))}
        orc.training_steps += 1
        orc.learn_batch(one_hot(b, A))
        steps += 1
    dt = time.perf_counter() - t0
    return dict(steps_per_s=steps / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for sarsa_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(shape)
        hst = host_rate(shape, d)
        g = gpu_rate(shape, d)
        res["shapes"][name] = dict(shape=shape, gpu=g, host_oracle=hst)
        print(f"{name}: GPU {g['steps_per_s']:.0f} gradient-steps/s ({g['launches_per_round']:.0f} launches/round) over "
              f"{g['window_s']:.1f} s; host eager-torch oracle {hst['steps_per_s']:.1f} steps/s ({hst['threads']} threads)")
        if name == "SARSA_method":
            op = on_policy(shape, d)
            res["shapes"]["on_policy"] = dict(shape=shape, gpu=op, host_oracle=hst)
            print(f"on_policy: GPU {op['learn_calls_per_s']:.0f} learn() calls/s over {op['window_s']:.1f} s, "
                  f"{op['episodes']} episodes, {op['graph_captures']} graph captures for {op['distinct_batch_sizes']} batch sizes; "
                  f"one capture {op['capture_ms']:.2f} ms, a replayed call {op['replay_call_ms']:.3f} ms; host eager-torch "
                  f"oracle {hst['steps_per_s']:.1f} steps/s (one step per learn())")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sarsa_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
