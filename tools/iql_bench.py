"""Developer tool: rates of the Implicit Q-Learning learner (pearl_b200.B200ImplicitQLearning) on one GPU, next to the
eager-torch restatement (oracle/iql_oracle.py) on the host:
  offline        Pearl's offline benchmark shape (benchmark_offline_rl.py: HalfCheetah obs 17, act 6 in [-1, 1],
                 VanillaContinuousActorNetwork, [256, 256] for all three nets, batch 256) on a 1e6-transition buffer:
                 gradient-steps/s of learn()
  IQL_online     IQL_online_method's shape (obs 4, 2 actions, [64, 64], batch 32): gradient-steps/s of learn()
  offline_batch  the offline shape through learn_batch() (what offline_learning() calls): calls/s, each call one round
                 on a batch already on the device, with its randint draw and the read-back of its three losses
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up; the launches
per round are the library's count.  Prints the card's name and power limit with the numbers.

    python tools/iql_bench.py [--out DIR]
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
from oracle.iql_oracle import OracleIQL  # noqa: E402

SHAPES = {"offline": dict(obs=17, act=6, A=None, hidden=256, B=256, n=1_000_000),
          "IQL_online": dict(obs=4, act=None, A=2, hidden=64, B=32, n=100_000)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(shape, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    n, obs = shape["n"], shape["obs"]
    d = dict(state=rng.standard_normal((n, obs), dtype=np.float32), next_state=rng.standard_normal((n, obs), dtype=np.float32),
             reward=rng.standard_normal(n, dtype=np.float32), term=rng.random(n) < 0.01)
    d["action"] = (rng.integers(0, shape["A"], size=n).astype(np.int32) if shape["A"]
                   else rng.uniform(-1.0, 1.0, size=(n, shape["act"])).astype(np.float32))
    return d


def act_kw(shape):
    return dict(n_actions=shape["A"]) if shape["A"] else dict(low=[-1.0] * shape["act"], high=[1.0] * shape["act"])


def learner(shape, rounds):
    h = shape["hidden"]
    return pearl_b200.B200ImplicitQLearning(state_dim=shape["obs"], actor_hidden_dims=[h, h], critic_hidden_dims=[h, h],
                                            value_critic_hidden_dims=[h, h], training_rounds=rounds, batch_size=shape["B"], seed=3,
                                            **act_kw(shape))


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


def gpu_rates(name, shape, d, rounds_per_call=200):
    n = shape["n"]
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    t = torch.from_numpy
    if shape["A"]:
        buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool),
                       max_number_actions=shape["A"])
    else:
        buf.is_action_continuous = True
        buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool))
    buf.seed(1)
    pl = learner(shape, rounds_per_call)
    trace = {}
    pl.learn(buf, trace=trace)                                  # warm-up: capture, module loads, algorithm choice
    out = {name: dict(launches_per_round=trace["launches"] / rounds_per_call)}
    rate, win = timed(lambda: pl.learn(buf), rounds_per_call)
    out[name].update(steps_per_s=rate, window_s=win)
    if name == "offline":
        rng = np.random.Generator(np.random.PCG64(7))
        batches = []
        for _ in range(64):
            i = rng.choice(n, size=shape["B"], replace=False)
            tt = lambda k: torch.from_numpy(d[k][i]).cuda()  # noqa: E731
            batches.append(pearl_b200.TransitionBatch(state=tt("state"), action=tt("action"), reward=tt("reward"),
                                                      next_state=tt("next_state"), terminated=tt("term")))
        k = [0]

        def one():
            pl.learn_batch(batches[k[0] % len(batches)])
            k[0] += 1
        for _ in range(8):
            one()                                               # warm-up of the learn_batch graph
        rate, win = timed(one, 1)
        out["offline_batch"] = dict(calls_per_s=rate, window_s=win)
    return out


def host_rate(shape, d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    h, B = shape["hidden"], shape["B"]
    orc = OracleIQL(shape["obs"], (h, h), (h, h), (h, h), **act_kw(shape))
    rng = np.random.Generator(np.random.PCG64(5))
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or steps < 3:
        i = rng.choice(shape["n"], size=B, replace=False)
        tt = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
        orc.learn_batch(dict(state=tt("state"), action=tt("action"), reward=tt("reward"), next_state=tt("next_state"),
                             terminated=tt("term")), rng.integers(0, 2, size=2))
        steps += 1
    dt = time.perf_counter() - t0
    return dict(steps_per_s=steps / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for iql_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(shape)
        hst = host_rate(shape, d)
        for k, g in gpu_rates(name, shape, d).items():
            res["shapes"][k] = dict(shape=shape, gpu=g, host_oracle=hst)
            rate = (f"{g['steps_per_s']:.0f} gradient-steps/s ({g['launches_per_round']:.0f} launches/round)" if "steps_per_s" in g
                    else f"{g['calls_per_s']:.0f} learn_batch calls/s")
            print(f"{k}: GPU {rate} over {g['window_s']:.1f} s; host eager-torch oracle {hst['steps_per_s']:.1f} steps/s "
                  f"({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "iql_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
