// Load-time weight re-layout: `.m` q40 blocks (18 B, file nibble order) -> device layout (common.cuh).
// Replaces the reference's host-side splitRow/ColMatmulWeight + per-socket streaming
// (src/nn/nn-core.cpp:289-322, src/nn/nn-network.cpp:830-888): the source may be a staging buffer on this
// GPU *or a peer GPU's staging buffer mapped over NVLink* — the kernel only sees (pointer, pitch, offset),
// so a worker can pull and re-tile its slice straight out of the root's memory.
#include "common.cuh"

namespace dl {

struct RepackArgs {
    const uint8_t *src;        // first byte of row 0 of the source matrix (raw 18-byte blocks)
    uint64_t srcRowPitch;      // bytes between consecutive source rows
    uint64_t srcColByteOffset; // byte offset of the first owned block inside a source row
    uint32_t rows;             // rows to convert
    uint32_t blocksPerRow;     // owned blocks per row
    uint32_t *dstQs;           // [dstRows][blocksPerRow*4]
    __half *dstScales;         // [dstRows][blocksPerRow]
    uint32_t dstRowStride;     // dst row = map(r) * dstRowStride + dstRowOffset
    uint32_t dstRowOffset;
    uint32_t headDim;          // != 0: rows are heads of this size stored half-split (NeoX); re-order each head
                               // to interleaved pairs so rotary pairs become adjacent rows (2j, 2j+1)
};

__global__ void __launch_bounds__(256) repackQ40Kernel(RepackArgs a) {
    const uint64_t total = (uint64_t)a.rows * a.blocksPerRow;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const uint32_t r = (uint32_t)(i / a.blocksPerRow);
        const uint32_t b = (uint32_t)(i % a.blocksPerRow);
        const uint8_t *s = a.src + (uint64_t)r * a.srcRowPitch + a.srcColByteOffset + (uint64_t)b * 18;
        uint8_t raw[18];
#pragma unroll
        for (int k = 0; k < 18; k++) raw[k] = s[k];
        // element e (0..31): e < 16 -> low nibble of byte e, else high nibble of byte e-16
        uint32_t words[4];
#pragma unroll
        for (int w = 0; w < 4; w++) {
            uint32_t word = 0;
#pragma unroll
            for (int slot = 0; slot < 8; slot++) {
                // slot order [e0,e2,e4,e6,e1,e3,e5,e7]
                const int eLocal = (slot < 4) ? (2 * slot) : (2 * (slot - 4) + 1);
                const int e = 8 * w + eLocal;
                const uint32_t nib = (e < 16) ? (raw[2 + e] & 0x0f) : (raw[2 + e - 16] >> 4);
                word |= nib << (4 * slot);
            }
            words[w] = word;
        }
        uint32_t rr = r;
        if (a.headDim) {
            const uint32_t h = r / a.headDim, j = r % a.headDim, half = a.headDim / 2;
            rr = h * a.headDim + (j < half ? 2 * j : 2 * (j - half) + 1);
        }
        const uint64_t dr = (uint64_t)rr * a.dstRowStride + a.dstRowOffset;
        uint4 *q = reinterpret_cast<uint4 *>(a.dstQs + (dr * a.blocksPerRow + b) * 4);
        *q = make_uint4(words[0], words[1], words[2], words[3]);
        const uint16_t sc = (uint16_t)raw[0] | ((uint16_t)raw[1] << 8);
        reinterpret_cast<uint16_t *>(a.dstScales)[dr * a.blocksPerRow + b] = sc;
    }
}

// Inverse (debug / tests): device layout -> f32 [rows][n]
__global__ void __launch_bounds__(256) dequantDeviceQ40Kernel(const uint32_t *qs, const __half *scales, uint32_t rows,
                                                              uint32_t blocksPerRow, float *out) {
    const uint64_t total = (uint64_t)rows * blocksPerRow;
    for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < total; i += (uint64_t)gridDim.x * blockDim.x) {
        const float d = __half2float(scales[i]);
        const uint4 q = *reinterpret_cast<const uint4 *>(qs + i * 4);
        const uint32_t w[4] = {q.x, q.y, q.z, q.w};
        float *o = out + i * 32;
#pragma unroll
        for (int k = 0; k < 4; k++)
#pragma unroll
            for (int s = 0; s < 4; s++) {
                const uint32_t t = (w[k] >> (4 * s)) & 0x000f000fu;
                o[8 * k + 2 * s] = (float)((int)(t & 0xf) - 8) * d;
                o[8 * k + 2 * s + 1] = (float)((int)(t >> 16) - 8) * d;
            }
    }
}

}  // namespace dl

DL_EXPORT int dl_repack_q40(const void *src, uint64_t srcRowPitch, uint64_t srcColByteOffset, uint32_t rows,
                            uint32_t blocksPerRow, void *dstQs, void *dstScales, uint32_t dstRowStride,
                            uint32_t dstRowOffset, uint32_t headDim, cudaStream_t stream) {
    dl::RepackArgs a{(const uint8_t *)src, srcRowPitch, srcColByteOffset, rows, blocksPerRow, (uint32_t *)dstQs,
                     (__half *)dstScales, dstRowStride, dstRowOffset, headDim};
    const uint64_t total = (uint64_t)rows * blocksPerRow;
    if (total == 0) return 0;
    const int grid = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    dl::repackQ40Kernel<<<grid, 256, 0, stream>>>(a);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}

DL_EXPORT int dl_dequant_device_q40(const void *qs, const void *scales, uint32_t rows, uint32_t blocksPerRow, float *out,
                                    cudaStream_t stream) {
    const uint64_t total = (uint64_t)rows * blocksPerRow;
    if (total == 0) return 0;
    const int grid = (int)((total + 255) / 256 < 132 * 16 ? (total + 255) / 256 : 132 * 16);
    dl::dequantDeviceQ40Kernel<<<grid, 256, 0, stream>>>((const uint32_t *)qs, (const __half *)scales, rows, blocksPerRow, out);
    DL_CUDA_CHECK(cudaGetLastError());
    return 0;
}
