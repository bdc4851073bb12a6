"""Developer tool: aggregate rate of the tensor-core learner group (R learners, `rounds` rounds) + phase stamps of CTA 0."""
import sys, os, time
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, ctypes as C
import pearl_b200
from pearl_b200 import _lib
from bench import Space, OBS, N_ACT, HIDDEN, BATCH
R = int(sys.argv[1]) if len(sys.argv) > 1 else 64
rounds = int(sys.argv[2]) if len(sys.argv) > 2 else 256
cap = int(sys.argv[3]) if len(sys.argv) > 3 else 100_000
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(1)
bufs, ls = [], []
for i in range(R):
    b = pearl_b200.B200ReplayBuffer(cap, rng="device")
    b.push_batch(torch.randn((cap, OBS), generator=g, device=dev), (torch.arange(cap, device=dev) % N_ACT).to(torch.int32),
                 torch.randn(cap, generator=g, device=dev), torch.randn((cap, OBS), generator=g, device=dev),
                 torch.rand(cap, generator=g, device=dev) < 0.02, torch.zeros(cap, dtype=torch.bool, device=dev), max_number_actions=N_ACT)
    b.seed(i + 1)
    bufs.append(b)
    ls.append(pearl_b200.B200DeepQLearning(state_dim=OBS, action_space=Space(N_ACT), hidden_dims=list(HIDDEN), training_rounds=rounds, batch_size=BATCH,
                                           action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(N_ACT),
                                           max_rounds_per_call=rounds, engine="tc").to(dev))
grp = pearl_b200.B200LearnerGroup(ls, bufs)
grp.set_kernel_timing(True)
for _ in range(2):
    grp.learn()
torch.cuda.synchronize()
t0 = time.perf_counter()
for _ in range(3):
    grp.learn()
torch.cuda.synchronize()
dt = (time.perf_counter() - t0) / 3
print(f"R={R} rounds={rounds}: {R*rounds/dt:.4e} steps/s wall; kernel {grp.last_kernel_ms():.2f} ms -> {R*rounds/grp.last_kernel_ms()*1e3:.4e} steps/s; {grp.last_kernel_ms()*1e3/rounds:.1f} us/round")
# phase stamps (single learner launch, unchunked)
st = torch.zeros((rounds, 16), dtype=torch.int64, device=dev)
_lib.check(ls[0]._libh.prl_dqn_set_profile(ls[0]._handle, C.c_void_p(st.data_ptr())))
grp.learn()
torch.cuda.synchronize()
s = st.cpu()[4:].double()
# stamps written by k_dqn_tc: 0 round start, 15 row scalars loaded (only the launch's first round loads its own), 1 soft
# update done, 2 target tiles loaded, 3 phase T done,
# 4 online small vectors loaded (and, before the W2^T tiles were kept in global memory, W2^T built), 5 tile 0 layer 1 done, 6 tile 0 forward / dZ2 / dH1 done, 8 weight gradients done,
# 7 gradients staged in shared memory, 10 AdamW sweep over W1 | b1 | W2 done, 9 small-parameter tail done (round end);
# in the weight-gradient passes of tile 0, rows 0-63: 11 dZ2^T / H1^T scattered, 12 dW2 / db2 waited for, 13 the operands
# of dW1s ready, 14 dW1s / [db1 | dW1a] waited for (the dW2 | db2 pass over rows 64-127 lies between 12 and 13)
phases = [("row scalars", 0, 15), ("soft target update", 15, 1), ("load target weights", 1, 2), ("phase T (layer 1 + all actions)", 2, 3),
          ("load online weights", 3, 4), ("tile 0: online layer 1", 4, 5), ("tile 0: fwd L2 + dZ2 + dH1", 5, 6),
          ("rest (weight grads, other tiles)", 6, 8), ("  tile 0 rows 0-63: dZ2^T / H1^T scatter", 6, 11),
          ("  tile 0 rows 0-63: dW2 / db2 products", 11, 12), ("  tile 0: to the operands of dW1s", 12, 13),
          ("  tile 0 rows 0-63: dW1s / [db1 | dW1a] products", 13, 14), ("AdamW: gradient staging", 8, 7),
          ("AdamW: sweep", 7, 10), ("AdamW: small-parameter tail", 10, 9)]
tot = (s[1:, 0] - s[:-1, 0]).mean()
print(f"{tot:.0f} clk/round (CTA {os.environ.get('PRL_TC_PROF_CTA', '0')} with {R} learners resident)")
for n, k, j in phases:
    print(f"  {n:46s} {(s[:, j]-s[:, k]).mean():10.0f} clk")
print(f"  {'AdamW (total)':46s} {(s[:, 9]-s[:, 8]).mean():10.0f} clk")
