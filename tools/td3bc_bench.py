"""Developer tool: rates of the TD3BC learner (pearl_b200.B200TD3BC) and of TD3's learn_batch on one GPU, next to the
eager-torch restatement (oracle/td3bc_oracle.py) on the host, at Pearl's offline benchmark shape (HalfCheetah obs 17,
act 6 in [-1, 1], [256, 256] actor, critics and behaviour network, batch 256, actor_update_freq 2):
  td3bc_learn   learn() over a 1e6-transition buffer: gradient-steps/s
  td3bc_batch   learn_batch() (what offline_learning() calls): calls/s, each call one round on a batch already on the
                device, with its noise draw and the read-back of its two losses; training steps alternate 0 / 1, so
                half the calls update the actor
  td3_batch     the same for TD3
The GPU rates come from CUDA events around whole calls, timed over windows of at least 2 s after a warm-up; the launches
per round are the library's count.  Prints the card's name and power limit with the numbers.

    python tools/td3bc_bench.py [--out DIR]
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
from pearl_b200.td3 import B200TD3, B200TD3BC  # noqa: E402
from oracle.td3bc_oracle import OracleTD3BC  # noqa: E402

OBS, ACT, H, B, N = 17, 6, 256, 256, 1_000_000


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    return dict(state=rng.standard_normal((N, OBS), dtype=np.float32), next_state=rng.standard_normal((N, OBS), dtype=np.float32),
                reward=rng.standard_normal(N, dtype=np.float32), term=rng.random(N) < 0.01,
                action=rng.uniform(-1.0, 1.0, size=(N, ACT)).astype(np.float32))


def learner(cls, rounds):
    kw = dict(behavior_hidden_dims=[H, H]) if cls is B200TD3BC else {}
    return cls(state_dim=OBS, low=[-1.0] * ACT, high=[1.0] * ACT, actor_hidden_dims=[H, H], critic_hidden_dims=[H, H],
               training_rounds=rounds, batch_size=B, seed=3, **kw)


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


def gpu_rates(d, rounds_per_call=200):
    t = torch.from_numpy
    buf = pearl_b200.B200ReplayBuffer(N, rng="device")
    buf.is_action_continuous = True
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(N, dtype=torch.bool))
    buf.seed(1)
    pl = learner(B200TD3BC, rounds_per_call)
    pl.learn(buf)                                               # warm-up: capture, module loads
    out = {"td3bc_learn": dict(launches_per_round=int(pl._lib.prl_td3_last_launches(pl._handle)) / rounds_per_call)}
    rate, win = timed(lambda: pl.learn(buf), rounds_per_call)
    out["td3bc_learn"].update(steps_per_s=rate, window_s=win)
    rng = np.random.Generator(np.random.PCG64(7))
    batches = []
    for _ in range(64):
        i = rng.choice(N, size=B, replace=False)
        tt = lambda k: torch.from_numpy(d[k][i]).cuda()  # noqa: E731
        batches.append(pearl_b200.TransitionBatch(state=tt("state"), action=tt("action"), reward=tt("reward"),
                                                  next_state=tt("next_state"), terminated=tt("term")))
    for name, cls in (("td3bc_batch", B200TD3BC), ("td3_batch", B200TD3)):
        pl = learner(cls, 1)
        k = [0]

        def one():
            pl._training_steps = k[0] % 2
            pl.learn_batch(batches[k[0] % len(batches)])
            k[0] += 1
        for _ in range(8):
            one()                                               # warm-up of both learn_batch graphs
        rate, win = timed(one, 1)
        out[name] = dict(calls_per_s=rate, window_s=win)
    return out


def host_rate(d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    orc = OracleTD3BC(OBS, ACT, (H, H), (H, H), [-1.0] * ACT, [1.0] * ACT, behavior_hidden=(H, H))
    rng = np.random.Generator(np.random.PCG64(5))
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or steps < 3:
        i = rng.choice(N, size=B, replace=False)
        tt = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
        orc.training_steps += 1
        orc.learn_batch(dict(state=tt("state"), action=tt("action"), reward=tt("reward"), next_state=tt("next_state"),
                             terminated=tt("term")), torch.randn(B, ACT) * 0.2)
        steps += 1
    dt = time.perf_counter() - t0
    return dict(steps_per_s=steps / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for td3bc_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shape": dict(obs=OBS, act=ACT, hidden=H, batch=B, n=N)}
    print("card:", res["card"])
    d = data()
    res["host_oracle"] = hst = host_rate(d)
    res["gpu"] = g = gpu_rates(d)
    for k, v in g.items():
        rate = (f"{v['steps_per_s']:.0f} gradient-steps/s ({v['launches_per_round']:.1f} launches/round)" if "steps_per_s" in v
                else f"{v['calls_per_s']:.0f} learn_batch calls/s")
        print(f"{k}: GPU {rate} over {v['window_s']:.1f} s")
    print(f"host eager-torch TD3BC oracle: {hst['steps_per_s']:.1f} steps/s ({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "td3bc_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
