// kvstate.cuh -- copy one session's KV-cache rows to other sessions of the same slice (b200_session_copy,
// b200_stream_fork).
#pragma once
#include "common.cuh"

namespace b200 {

constexpr uint32_t kFanChunk = 32768;                 // bytes per stage; two stages per CTA
constexpr int kFanSmem = 2 * kFanChunk;

// Rows [0, n_keep) of every layer's K and V plane, from session src to the n_dst sessions dsts[], in one launch.
// blockIdx.y is the plane (layer * 2 + {0 K, 1 V}); CTA x takes the plane's chunks x, x + gridDim.x, ...  Each chunk
// crosses HBM once inward (a TMA load into shared memory) and n_dst times outward (one bulk store per destination), so a
// source byte is read once however many destinations there are.  Two stages: chunk i's load lands while chunk i - 1's
// stores still read the other stage.  A plane's rows are contiguous (n_keep * E * 2 bytes, a multiple of 64 since
// E % 32 == 0) and every plane starts at a multiple of n_ctx * E * 2 bytes, so every bulk copy is 16-byte aligned.
// One thread issues everything: the copy engine moves the bytes.
__global__ void __launch_bounds__(32) k_kv_fanout(uint16_t * kc, uint16_t * vc, size_t sess_stride, size_t plane_stride,
                                                  int src, const int * __restrict__ dsts, int n_dst, uint32_t plane_bytes) {
    extern __shared__ __align__(128) uint8_t stage[];
    __shared__ uint64_t full[2];
    if (threadIdx.x != 0) return;
    uint8_t * base = (uint8_t *) ((blockIdx.y & 1) ? vc : kc) + (size_t) (blockIdx.y >> 1) * plane_stride * 2;
    const uint8_t * from = base + (size_t) src * sess_stride * 2;
    const uint32_t n_chunks = (plane_bytes + kFanChunk - 1) / kFanChunk;
    uint32_t c = blockIdx.x;
    if (c >= n_chunks) return;
    mbar_init(&full[0], 1); mbar_init(&full[1], 1);
    mbar_fence_init();
    auto load = [&](uint32_t chunk, int st) {
        const uint32_t bytes = min(kFanChunk, plane_bytes - chunk * kFanChunk);
        mbar_arrive_expect_tx(&full[st], bytes);
        bulk_g2s(stage + st * kFanChunk, from + (size_t) chunk * kFanChunk, bytes, &full[st]);
    };
    load(c, 0);
    for (uint32_t i = 0; c < n_chunks; i++, c += gridDim.x) {
        const int st = i & 1;
        const uint32_t bytes = min(kFanChunk, plane_bytes - c * kFanChunk);
        mbar_wait(&full[st], (i >> 1) & 1);
        for (int d = 0; d < n_dst; d++)
            s2g(base + (size_t) dsts[d] * sess_stride * 2 + (size_t) c * kFanChunk, stage + st * kFanChunk, bytes);
        bulk_commit();
        if (c + gridDim.x < n_chunks) {
            bulk_wait_read<1>();                       // chunk i - 1's stores have read the other stage
            load(c + gridDim.x, st ^ 1);
        }
    }
    bulk_wait<0>();
}

}  // namespace b200
