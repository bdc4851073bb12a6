"""Developer tool: time the learners' contraction shapes on the SIMT tiles and on the wgmma tiles (CUDA events around
replays of a CUDA graph of 20 launches, so the figure is the device-side issue-to-issue time — what the CUDA-graph
replay of a learner round sees).  python tools/gemm_bench.py [reps]"""
import ctypes as C
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from pearl_b200 import _lib  # noqa: E402


def p(t):
    return C.c_void_p(t.data_ptr()) if t is not None else None


def main():
    reps = int(sys.argv[1]) if len(sys.argv) > 1 else 200
    lib = _lib.init(0)
    dev = "cuda"
    shapes = [  # (name, op, M, N, K, nets)
        ("SAC fwd L1 512x256x376", 0, 512, 256, 376, 1),
        ("SAC fwd twin-critic L1 512x256x393 x2", 0, 512, 256, 393, 2),
        ("SAC fwd L2 512x256x256", 0, 512, 256, 256, 1),
        ("SAC head 512x17x256", 0, 512, 17, 256, 1),
        ("SAC q head 512x1x256 x2", 0, 512, 1, 256, 2),
        ("SAC bwd-x 512x256->256", 1, 512, 256, 256, 1),
        ("SAC bwd-w 256x376 over 512", 2, 512, 256, 376, 1),
        ("SAC bwd-w twin 256x393 over 512 x2", 2, 512, 256, 393, 2),
        ("PPO fwd L1 256x64x210", 0, 256, 64, 210, 1),
        ("PPO fwd L2 256x64x64", 0, 256, 64, 64, 1),
        ("PPO bwd-w 64x210 over 256", 2, 256, 64, 210, 1),
        ("PPO preprocess 8192x64x210", 0, 8192, 64, 210, 1),
        ("PPO preprocess 8192x256x210", 0, 8192, 256, 210, 1),
        ("big 65536x256x256", 0, 65536, 256, 256, 1),
    ]
    for name, op, M, N, K, nets in shapes:
        a = torch.randn((nets, M, K if op == 0 else N), device=dev)
        b = torch.randn((nets, N, K), device=dev) if op != 2 else torch.randn((nets, M, K), device=dev)
        bias = torch.randn((nets, N), device=dev) if op == 0 else None
        c = torch.empty((nets, M, N) if op == 0 else ((nets, M, K) if op == 1 else (nets, N, K)), device=dev)
        ct = torch.empty((nets, N), device=dev) if op == 2 else None
        flops = 2.0 * M * N * K * nets
        out = []
        for engine in (0, 64, 164, 132):
            side = torch.cuda.Stream()
            sp = C.c_void_p(side.cuda_stream)

            def run():
                _lib.check(lib.prl_test_contraction(op, engine, M, N, K, p(a), p(b), None, 0, p(bias), None, 1 if op == 0 else 0, 0,
                                                    p(c), p(ct), nets, sp))
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for _ in range(3):
                    run()
                side.synchronize()
                graph = torch.cuda.CUDAGraph()       # 20 launches per replay: device-side issue-to-issue time, no host in the loop
                with torch.cuda.graph(graph, stream=side):
                    for _ in range(20):
                        run()
                graph.replay()
                side.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(side)
                for _ in range(max(reps // 20, 1)):
                    graph.replay()
                e1.record(side)
                side.synchronize()
            us = e0.elapsed_time(e1) * 1e3 / (max(reps // 20, 1) * 20)
            out.append(f"{['simt', 'ss64', 'ts64', 'ts32'][(0, 64, 164, 132).index(engine)]} {us:7.2f} us ({flops / us * 1e-6:7.2f} TF/s)")
        print(f"{name:42s} " + "  ".join(out), flush=True)


if __name__ == "__main__":
    main()
