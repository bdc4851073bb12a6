"""Developer tool: phase breakdown (SM clocks of CTA 0) of the tensor-core learner kernel."""
import sys, os
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch, ctypes as C
import pearl_b200
from pearl_b200 import _lib
from bench import Space, OBS, N_ACT, HIDDEN, BATCH
rounds = 64
dev = torch.device("cuda", 0)
g = torch.Generator(device=dev).manual_seed(1)
cap = 200_000
b = pearl_b200.B200ReplayBuffer(cap, rng="device")
b.push_batch(torch.randn((cap, OBS), generator=g, device=dev), (torch.arange(cap, device=dev) % N_ACT).to(torch.int32),
             torch.randn(cap, generator=g, device=dev), torch.randn((cap, OBS), generator=g, device=dev),
             torch.rand(cap, generator=g, device=dev) < 0.02, torch.zeros(cap, dtype=torch.bool, device=dev), max_number_actions=N_ACT)
b.seed(1)
L = pearl_b200.B200DeepQLearning(state_dim=OBS, action_space=Space(N_ACT), hidden_dims=list(HIDDEN), training_rounds=rounds, batch_size=BATCH,
                                 action_representation_module=pearl_b200.OneHotActionTensorRepresentationModule(N_ACT),
                                 max_rounds_per_call=rounds, engine="tc").to(dev)
L.learn(b)
st = torch.zeros((rounds, 16), dtype=torch.int64, device=dev)
_lib.check(L._libh.prl_dqn_set_profile(L._handle, C.c_void_p(st.data_ptr())))
L.set_kernel_timing(True)
L.learn(b)
ms = L.last_kernel_ms()
s = st.cpu()[4:].double()
# stamps written by k_dqn_tc (see tools/tc_bench.py): AdamW is split into gradient staging (8 -> 7), the sweep over
# W1 | b1 | W2 (7 -> 10) and the small-parameter tail (10 -> 9)
phases = [("row scalars + soft upd", 0, 1), ("load target weights", 1, 2), ("phase T (layer 1 + all actions)", 2, 3),
          ("load online weights + W2^T", 3, 4), ("tile 0: online layer 1", 4, 5), ("tile 0: fwd L2 + dZ2 + dH1", 5, 6),
          ("rest (weight grads, other tiles)", 6, 8), ("AdamW: gradient staging", 8, 7), ("AdamW: sweep", 7, 10),
          ("AdamW: small-parameter tail", 10, 9)]
tot = (s[1:, 0] - s[:-1, 0]).mean()
print(f"kernel {ms*1e3/rounds:.1f} us/round; {tot:.0f} clk/round")
for n, k, j in phases:
    print(f"  {n:36s} {(s[:, j]-s[:, k]).mean():10.0f} clk")
