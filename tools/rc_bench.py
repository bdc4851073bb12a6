"""Developer tool: agent.learn()-equivalent calls per second of TD3 with Pearl's reward-constrained safety module on one GPU,
next to TD3 alone and the eager-torch restatement (oracle/rc_safety_oracle.py) on the host, at Pearl's RCTD3 shape
(utils/scripts/benchmark_config.py RCTD3_method_const_*: obs 17, act 6 in [-1, 1], [256, 256] actor, critics and cost
critics, batch 256, training_rounds 1, constraint 0.2, lr_lambda 1e-3, upper bound 200):
  td3         B200TD3.learn() alone: one round per call (no multiplier)
  td3_rc      one round on cost-shaped rewards + the CUDA cost-critic and lambda step, with its read-back of lambda
  host_oracle the same call in eager torch on the host
The GPU rates come from CUDA events around whole calls over windows of at least 2 s after a warm-up; the launches per
call are the library's counts.  Prints the card's name and power limit with the numbers.

    python tools/rc_bench.py [--out DIR]
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
from pearl_b200.rc_safety import B200RCSafetyModule  # noqa: E402
from pearl_b200.td3 import B200TD3  # noqa: E402
from oracle.rc_safety_oracle import OracleCostCritic, agent_learn  # noqa: E402
from oracle.td3_oracle import OracleTD3  # noqa: E402

OBS, ACT, H, B, N = 17, 6, 256, 256, 200_000
RC = dict(constraint_value=0.2, lr_lambda=1e-3, lambda_constraint_ub_value=200.0)


def card() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:   # noqa: BLE001
        return f"nvidia-smi unavailable ({e})"


def data(seed=0):
    rng = np.random.Generator(np.random.PCG64(seed))
    return dict(state=rng.standard_normal((N, OBS), dtype=np.float32), next_state=rng.standard_normal((N, OBS), dtype=np.float32),
                reward=rng.standard_normal(N, dtype=np.float32), terminated=rng.random(N) < 0.01,
                action=rng.uniform(-1.0, 1.0, size=(N, ACT)).astype(np.float32), cost=rng.uniform(0.0, 1.0, N).astype(np.float32))


def timed(fn, window_s=2.0):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    done, ms = 0, 0.0
    while ms < window_s * 1e3:
        e0.record()
        for _ in range(50):
            fn()
        e1.record()
        e1.synchronize()
        ms += e0.elapsed_time(e1)
        done += 50
    return done / (ms / 1e3), ms / 1e3


def gpu_rates(d):
    t = torch.from_numpy
    buf = pearl_b200.B200ReplayBuffer(N, rng="device")
    buf.is_action_continuous = True
    buf.push_batch(t(d["state"]), t(d["action"]), t(d["reward"]), t(d["next_state"]), t(d["terminated"]), torch.zeros(N, dtype=torch.bool),
                   cost=t(d["cost"]))
    buf.seed(1)
    out = {}
    for name, with_rc in (("td3", False), ("td3_rc", True)):
        pl = B200TD3(state_dim=OBS, low=[-1.0] * ACT, high=[1.0] * ACT, actor_hidden_dims=[H, H], critic_hidden_dims=[H, H],
                     training_rounds=1, batch_size=B, seed=3)
        rc = B200RCSafetyModule(state_dim=OBS, low=[-1.0] * ACT, high=[1.0] * ACT, critic_hidden_dims=[H, H], batch_size=B, seed=4, **RC)
        if with_rc:
            pl.safety_module = rc

        def call():
            pl.learn(buf)
            if with_rc:
                rc.learn(buf, pl)
        for _ in range(4):
            call()                                                # warm-up: captures, module loads
        launches = int(pl._lib.prl_td3_last_launches(pl._handle)) + (rc.last_launches if with_rc else 0)
        rate, win = timed(call)
        out[name] = dict(calls_per_s=rate, window_s=win, launches_per_call=launches)
        if with_rc:
            out[name]["lambda_after"] = rc.lambda_constraint
    return out


def host_rate(d, window_s=2.0):
    torch.set_num_threads(os.cpu_count() or 1)
    orc = OracleTD3(OBS, ACT, (H, H), (H, H), [-1.0] * ACT, [1.0] * ACT)
    cc = OracleCostCritic(OBS, ACT, (H, H), constraint=RC["constraint_value"], lr_lambda=RC["lr_lambda"], ub=RC["lambda_constraint_ub_value"])
    rng = np.random.Generator(np.random.PCG64(5))
    calls, t0 = 0, time.perf_counter()
    while time.perf_counter() - t0 < window_s or calls < 3:
        rows = []
        for _ in range(2):
            i = rng.choice(N, size=B, replace=False)
            rows.append({k: torch.from_numpy(v[i]) for k, v in d.items()})
        agent_learn(orc, cc, rows, 1, torch.randn(1, B, ACT) * 0.2)
        calls += 1
    dt = time.perf_counter() - t0
    return dict(calls_per_s=calls / dt, window_s=dt, threads=torch.get_num_threads())


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default=None, help="directory for rc_bench.json")
    args = ap.parse_args()
    res = {"card": card(), "shape": dict(obs=OBS, act=ACT, hidden=H, batch=B, n=N, training_rounds=1, **RC)}
    print("card:", res["card"])
    d = data()
    res["gpu"] = g = gpu_rates(d)
    res["host_oracle"] = hst = host_rate(d)
    for k, v in g.items():
        print(f"{k}: GPU {v['calls_per_s']:.0f} agent.learn() calls/s ({v['launches_per_call']} launches/call) over {v['window_s']:.1f} s")
    print(f"host eager-torch oracle (TD3 round + RC step): {hst['calls_per_s']:.1f} calls/s ({hst['threads']} threads)")
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "rc_bench.json"), "w") as f:
            json.dump(res, f, indent=1)


if __name__ == "__main__":
    main()
