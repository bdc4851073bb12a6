"""Developer tool: gradient-steps/s of the discrete SAC learner (pearl_b200.B200SoftActorCritic) on one GPU, next to the
eager-torch restatement (oracle/sac_discrete_oracle.py) on the host, at two shapes:
  SAC_method  Pearl's benchmark configuration (obs 4, 2 actions, [64, 64], batch 32)
  stress      obs 128, 16 actions, [256, 256], batch 256, dynamic next-action sets
The GPU rate comes from CUDA events around whole learn() calls, timed over windows of at least 2 s after a warm-up call;
the launches per round are the library's count.  Prints the card's name and power limit with the numbers.

    python tools/sacd_bench.py [--out DIR]
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
from oracle.sac_discrete_oracle import OracleSACDiscrete  # noqa: E402

SHAPES = {"SAC_method": dict(obs=4, A=2, hidden=64, B=32, dynamic=False),
          "stress": dict(obs=128, A=16, hidden=256, B=256, dynamic=True)}


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(n, obs, A, dynamic, seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    ids = np.tile(np.arange(A, dtype=np.uint8), (n, 1))
    cnt = np.full(n, A, dtype=np.int32)
    if dynamic:
        cnt = rng.integers(1, A + 1, size=n).astype(np.int32)
        for i in range(n):
            ids[i, :] = 0
            ids[i, :cnt[i]] = np.sort(rng.choice(A, size=cnt[i], replace=False))
    return dict(state=rng.standard_normal((n, obs)).astype(np.float32), next_state=rng.standard_normal((n, obs)).astype(np.float32),
                reward=rng.standard_normal(n).astype(np.float32), action=rng.integers(0, A, size=n).astype(np.int32),
                term=rng.random(n) < 0.02, ids=ids, cnt=cnt)


def gpu_rate(shape, d, rounds_per_call=200, window_s=2.0):
    n = d["state"].shape[0]
    buf = pearl_b200.B200ReplayBuffer(n, rng="device")
    t = torch.from_numpy
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["term"]), torch.zeros(n, dtype=torch.bool),
                   next_available_ids=t(d["ids"]) if shape["dynamic"] else None,
                   next_available_count=t(d["cnt"]) if shape["dynamic"] else None, max_number_actions=shape["A"])
    buf.seed(1)
    h = shape["hidden"]
    pl = pearl_b200.B200SoftActorCritic(state_dim=shape["obs"], n_actions=shape["A"], actor_hidden_dims=[h, h], critic_hidden_dims=[h, h],
                                        training_rounds=rounds_per_call, batch_size=shape["B"], entropy_coef=0.1, seed=3)
    trace = {}
    pl.learn(buf, trace=trace)                                  # warm-up: capture, module loads, algorithm choice
    launches = trace["launches"] / rounds_per_call
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    steps, ms = 0, 0.0
    while ms < window_s * 1e3:
        e0.record()
        rep = pl.learn(buf)
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        steps += rounds_per_call
    return dict(steps_per_s=steps / (ms / 1e3), window_s=ms / 1e3, launches_per_round=launches,
                last_actor_loss=rep["actor_loss"][-1], last_critic_loss=rep["critic_loss"][-1])


def host_rate(shape, d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    h, B, A = shape["hidden"], shape["B"], shape["A"]
    orc = OracleSACDiscrete(shape["obs"], A, (h, h), (h, h), entropy_coef=0.1)
    rng = np.random.Generator(np.random.PCG64(5))
    n = d["state"].shape[0]
    steps, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or steps < 3:
        i = rng.choice(n, size=B, replace=False)
        tt = lambda k: torch.from_numpy(d[k][i])  # noqa: E731
        orc.learn_batch(dict(state=tt("state"), action=tt("action"), reward=tt("reward"), next_state=tt("next_state"), terminated=tt("term"),
                             next_ids=tt("ids").long(), next_mask=torch.arange(A).unsqueeze(0) >= tt("cnt").unsqueeze(1)))
        steps += 1
    dt = time.perf_counter() - t0
    return dict(steps_per_s=steps / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for sacd_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shapes": {}}
    print("card:", res["card"])
    for name, shape in SHAPES.items():
        d = data(50_000, shape["obs"], shape["A"], shape["dynamic"])
        g, hst = gpu_rate(shape, d), host_rate(shape, d)
        res["shapes"][name] = dict(shape=shape, gpu=g, host_oracle=hst)
        print(f"{name}: GPU {g['steps_per_s']:.0f} gradient-steps/s ({g['launches_per_round']:.0f} launches/round, {g['window_s']:.1f} s), "
              f"host eager-torch oracle {hst['steps_per_s']:.1f} steps/s ({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "sacd_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
