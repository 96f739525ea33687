// Speculative decoding with a draft model: the device half of one round (engine.cu: dl_spec_round).
//
// A round starts from the last emitted token t at position p, held in the target's tokens[0] / pos[0]. The draft runs k + 1 greedy
// steps from (t, p) and hands its tokens d1..dk to the target's rows 1..k; the target verifies [t, d1..dk] at p..p+k as one batched
// forward whose logits GEMV ends in a per-row arg-max g0..gk; the accept kernel below keeps the longest agreeing prefix.
#include "kernels.h"

namespace dl {

// Start of a round: the draft continues from the target's (token, position) and the target's rows 1..k get positions p+1..p+k.
__global__ void specStageKernel(SpecAcceptArgs a) {
    const int i = threadIdx.x;
    const int p = a.targetPos[0];
    if (i >= 1 && i <= (int)a.k) a.targetPos[i] = p + i;
    if (i == 0) {
        a.draftTokens[0] = a.targetTokens[0];
        a.draftPos[0] = p;
    }
}

// a = the longest prefix with d(i+1) == g(i); the round emits d1..da and the correction g(a), i.e. g(0..a). One warp.
__global__ void specAcceptKernel(SpecAcceptArgs a) {
    const int lane = threadIdx.x;
    const int p = a.targetPos[0];
    const uint32_t k = a.k;
    // lane i (< k) agrees when the draft's token i + 1 equals the target's choice after row i
    const bool agree = (uint32_t)lane < k && a.targetTokens[lane + 1] == a.verifyTokens[lane];
    const uint32_t disagree = __ballot_sync(0xffffffffu, !agree);
    const uint32_t acc = (uint32_t)(__ffs(disagree) - 1);   // lane k never agrees, so acc <= k
    if ((uint32_t)lane <= acc) {
        const int tok = a.verifyTokens[lane];
        const int q = p + 1 + lane;
        a.result[kSpecResultHead + lane] = tok;
        if (a.targetHistory && (uint32_t)q < a.historyCap) a.targetHistory[q] = tok;
        if (a.draftHistory && (uint32_t)q < a.draftHistoryCap) a.draftHistory[q] = tok;
    }
    if (lane == 0) {
        const int last = a.verifyTokens[acc];
        a.result[0] = (int)acc;
        a.result[1] = (int)acc + 1;
        a.result[2] = (int)k;
        a.result[3] = p + (int)acc + 1;
        a.targetTokens[0] = last;
        a.targetPos[0] = p + (int)acc + 1;
        a.draftTokens[0] = last;
        a.draftPos[0] = p + (int)acc + 1;
    }
}

int launchSpecStage(const SpecAcceptArgs &a, cudaStream_t stream) {
    if (a.k < 1 || a.k > kSpecMaxDraft) return -1;
    specStageKernel<<<1, 32, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

int launchSpecAccept(const SpecAcceptArgs &a, cudaStream_t stream) {
    if (a.k < 1 || a.k > kSpecMaxDraft) return -1;
    specAcceptKernel<<<1, 32, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

}  // namespace dl

// Accept kernel on explicit device buffers (tests/test_gpu_speculative.py): verifyTokens [k + 1] are the target's arg-maxes,
// targetTokens [k + 1] hold t, d1..dk and targetPos[0] = p; result [kSpecResultWords]. History pointers may be null.
DL_EXPORT int dl_spec_accept(const int *verifyTokens, int *targetTokens, int *targetPos, int *targetHistory, uint32_t historyCap,
                             int *draftTokens, int *draftPos, int *draftHistory, uint32_t draftHistoryCap, uint32_t k, int *result,
                             cudaStream_t stream) {
    dl::SpecAcceptArgs a{};
    a.verifyTokens = verifyTokens; a.targetTokens = targetTokens; a.targetPos = targetPos; a.targetHistory = targetHistory;
    a.historyCap = historyCap; a.draftTokens = draftTokens; a.draftPos = draftPos; a.draftHistory = draftHistory;
    a.draftHistoryCap = draftHistoryCap; a.k = k; a.result = result;
    return dl::launchSpecAccept(a, stream);
}
