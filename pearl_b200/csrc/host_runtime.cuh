// host_runtime.cuh — host-side plumbing shared by the learners: torch's AdamW step scalars, the pinned staging of a
// per-call block, CUDA-graph capture of one round and workspace carving.  No device code.
#pragma once
#include <math.h>

#include "common.cuh"

namespace prl {

// torch.optim.AdamW's scalars of optimizer step `step`, evaluated in double as Python does and rounded to fp32:
// (lr / (1 - beta1^step), sqrt(1 - beta2^step)), the `scal` entry k_adamw (gemm.cuh) and k_dqn_learn read per round
inline float2 adam_scal(double lr, double beta1, double beta2, int64_t step) {
    const double t = (double)step;
    const double bc1 = 1.0 - pow(beta1, t), bc2 = 1.0 - pow(beta2, t);
    return make_float2((float)(lr / bc1), (float)sqrt(bc2));
}

// Two pinned host buffers, each with an event recorded after the copy that reads it: the host fills one while the copy
// out of the other may still be in flight.  close() is safe on a stage never opened or partly opened.
struct Stage {
    char *host[2] = {nullptr, nullptr};
    cudaEvent_t done[2] = {nullptr, nullptr};
    int next = 0;

    // on failure, what was made is released again
    cudaError_t open(size_t bytes) {
        for (int i = 0; i < 2; i++) {
            cudaError_t e = cudaHostAlloc((void **)&host[i], bytes, cudaHostAllocDefault);
            if (e == cudaSuccess) e = cudaEventCreateWithFlags(&done[i], cudaEventDisableTiming);
            if (e != cudaSuccess) { close(); return e; }
        }
        return cudaSuccess;
    }
    void close() {
        for (int i = 0; i < 2; i++) {
            if (done[i]) { cudaEventSynchronize(done[i]); cudaEventDestroy(done[i]); }
            if (host[i]) cudaFreeHost(host[i]);
            host[i] = nullptr; done[i] = nullptr;
        }
    }
    // the buffer to fill next, once the copy that last read it has finished
    template <class T>
    int wait(T **h) {
        PRL_CUDA(cudaEventSynchronize(done[next]));
        *h = reinterpret_cast<T *>(host[next]);
        return PRL_OK;
    }
    // copies the first `bytes` of the buffer wait() returned to `dev` on `st`
    int send(void *dev, size_t bytes, cudaStream_t st) {
        PRL_CUDA(cudaMemcpyAsync(dev, host[next], bytes, cudaMemcpyHostToDevice, st));
        PRL_CUDA(cudaEventRecord(done[next], st));
        next ^= 1;
        return PRL_OK;
    }
};

// Records round(stream) into *exec, replacing the graph *exec held, on a non-blocking stream in thread-local capture mode.
// *exec is null on failure.  A failure of the round itself is returned once the capture has been ended.
template <class Round>
int capture_graph(cudaGraphExec_t *exec, const char *who, Round &&round) {
    if (*exec) { cudaGraphExecDestroy(*exec); *exec = nullptr; }
    cudaStream_t cs;
    PRL_CUDA(cudaStreamCreateWithFlags(&cs, cudaStreamNonBlocking));
    cudaGraph_t graph = nullptr;
    int rc = PRL_OK;
    cudaError_t e = cudaStreamBeginCapture(cs, cudaStreamCaptureModeThreadLocal);
    if (e == cudaSuccess) {
        rc = round(cs);
        e = cudaStreamEndCapture(cs, &graph);
    }
    if (e == cudaSuccess && rc == PRL_OK) e = cudaGraphInstantiate(exec, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    cudaStreamDestroy(cs);
    if (rc == PRL_OK && e == cudaSuccess) return PRL_OK;
    *exec = nullptr;
    return rc != PRL_OK ? rc : fail(PRL_ECUDA, "%s: graph capture failed: %s", who, cudaGetErrorString(e));
}

// One list that both sizes and assigns a workspace: every buffer starts 256-byte aligned, right after the previous one.
// With a null base only `bytes` counts (the *_workspace_bytes figure); with the caller's workspace the pointers are set.
struct Carve {
    char *base;
    int64_t bytes = 0;
    template <class T>
    void operator()(T *&p, int64_t count) {
        p = base ? reinterpret_cast<T *>(base + bytes) : nullptr;
        bytes = (bytes + count * (int64_t)sizeof(T) + 255) / 256 * 256;
    }
};

}  // namespace prl
