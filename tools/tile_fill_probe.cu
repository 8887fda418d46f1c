// Tile fill probe: the stage loop of the regex / delimiter kernels' line loader (TdfaLoader in
// loongcollector_b200/csrc/lc_kernels.cu) alone, with two layouts of the per-warp 4 KB staging tile.
//
//   chunk-major  slot(line, q) = q * 512 + ((line ^ q) << 4)            one LDGSTS writes 32 different 128-byte rows
//   line-major   slot(line, q) = line * 128 + (((q ^ line) & 7) << 4)   one LDGSTS writes 4 rows, one per global line
//
// 1024-thread blocks, one per SM; every warp claims 32-line batches (lines of `pitch` bytes, 16 chunks each) and
// runs per stage of 8 chunks: 8 cp.async of 16 B per lane, wait, __syncwarp, one LDS.128 per lane and chunk folded
// into an XOR that is written out at the end.  Prints "layout placement working_set_mb reps t0 t1 ..." (ms).
//
//   tile_fill_probe <lines> <pitch> <reps> <working-set lines>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <vector>

#include <cuda_runtime.h>

#define CK(x)                                                                                                          \
    do {                                                                                                               \
        cudaError_t e_ = (x);                                                                                          \
        if (e_ != cudaSuccess) {                                                                                       \
            fprintf(stderr, "%s:%d %s\n", __FILE__, __LINE__, cudaGetErrorString(e_));                                 \
            exit(1);                                                                                                   \
        }                                                                                                              \
    } while (0)

__device__ __forceinline__ uint2 lds_u64_v(uint32_t a) {
    uint2 v;
    asm volatile("ld.shared.v2.u32 {%0, %1}, [%2];" : "=r"(v.x), "=r"(v.y) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ uint4 lds_u128_v(uint32_t a) {
    uint4 v;
    asm volatile("ld.shared.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(v.x), "=r"(v.y), "=r"(v.z), "=r"(v.w) : "r"(a) : "memory");
    return v;
}
__device__ __forceinline__ void sts_u64(uint32_t a, uint32_t x, uint32_t y) {
    asm volatile("st.shared.v2.u32 [%0], {%1, %2};" ::"r"(a), "r"(x), "r"(y) : "memory");
}
__device__ __forceinline__ void cp_async_16(uint32_t dst, const void* src) {
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(dst), "l"(src) : "memory");
}
__device__ __forceinline__ void cp_async_wait_all() {
    asm volatile("cp.async.commit_group;\n\tcp.async.wait_group 0;" ::: "memory");
}

template <bool LINE_MAJOR>
__device__ __forceinline__ uint32_t slot(uint32_t tile, uint32_t line, uint32_t q) {
    return LINE_MAJOR ? tile + line * 128 + (((q ^ line) & 7) << 4) : tile + (q << 9) + ((line ^ q) << 4);
}

template <bool LINE_MAJOR>
__global__ void __launch_bounds__(1024, 1)
    fill_kernel(const uint4* __restrict__ g, uint32_t lines, uint32_t pitch16, uint32_t first16, uint32_t ws_lines,
                uint32_t* __restrict__ out) {
    extern __shared__ uint4 smem[];
    const uint32_t lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nwarps = blockDim.x >> 5;
    const uint32_t s0abs = (uint32_t)__cvta_generic_to_shared(smem);
    const uint32_t info_abs = s0abs + wid * 256, tile_abs = s0abs + nwarps * 256 + wid * 4096;
    const uint32_t ld_q = lane & 7, ld_L0 = (lane >> 3) * 8, ld_info = info_abs + ld_L0 * 8;
    uint32_t acc = 0;
    for (uint32_t b = (blockIdx.x * nwarps + wid) * 32; b < lines; b += gridDim.x * nwarps * 32) {
        const uint32_t line = b + lane;
        sts_u64(info_abs + lane * 8, (line % ws_lines) * pitch16 + first16, line < lines ? 16u : 0u);
        __syncwarp();
        for (uint32_t s0 = 0; s0 < 16; s0 += 8) {
            const uint32_t cidx = s0 + ld_q;
#pragma unroll
            for (uint32_t r = 0; r < 8; ++r) {
                const uint2 inf = lds_u64_v(ld_info + r * 8);
                if (cidx < inf.y)
                    cp_async_16(slot<LINE_MAJOR>(tile_abs, ld_L0 + r, ld_q), g + inf.x + cidx);
            }
            cp_async_wait_all();
            __syncwarp();
#pragma unroll
            for (uint32_t q = 0; q < 8; ++q) {
                const uint4 v = lds_u128_v(slot<LINE_MAJOR>(tile_abs, lane, q));
                acc ^= v.x ^ v.y ^ v.z ^ v.w;
            }
            __syncwarp();
        }
    }
    out[blockIdx.x * blockDim.x + threadIdx.x] = acc;
}

int main(int argc, char** argv) {
    if (argc != 5) {
        fprintf(stderr, "usage: %s <lines> <pitch> <reps> <working-set lines>\n", argv[0]);
        return 2;
    }
    const uint32_t lines = (uint32_t)atoi(argv[1]), pitch = (uint32_t)atoi(argv[2]), reps = (uint32_t)atoi(argv[3]);
    const uint32_t ws_lines = (uint32_t)atoi(argv[4]);
    if (pitch % 16 || pitch < 256 || ws_lines == 0 || ws_lines > lines) {
        fprintf(stderr, "pitch must be a multiple of 16 and >= 256; 0 < working set <= lines\n");
        return 2;
    }
    int dev = 0, sms = 0;
    CK(cudaSetDevice(dev));
    CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev));
    const size_t bytes = (size_t)lines * pitch + 256;
    uint4* d = nullptr;
    uint32_t* out = nullptr;
    CK(cudaMalloc(&d, bytes));
    CK(cudaMemset(d, 0x5A, bytes));
    const uint32_t threads = 1024, smem = 32 * (256 + 4096);
    CK(cudaMalloc(&out, (size_t)sms * threads * 4));
    CK(cudaFuncSetAttribute(fill_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    CK(cudaFuncSetAttribute(fill_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
    cudaEvent_t e0, e1;
    CK(cudaEventCreate(&e0));
    CK(cudaEventCreate(&e1));
    // placements: line starts 128-byte aligned (one global line per stage), and 16 bytes in (every stage straddles two)
    for (uint32_t first16 : {0u, 1u}) {
        std::vector<float> t[2];
        auto launch = [&](int lm) {
            if (lm)
                fill_kernel<true><<<sms, threads, smem>>>(d, lines, pitch / 16, first16, ws_lines, out);
            else
                fill_kernel<false><<<sms, threads, smem>>>(d, lines, pitch / 16, first16, ws_lines, out);
        };
        for (int w = 0; w < 3; ++w)
            for (int lm = 0; lm < 2; ++lm)
                launch(lm);
        CK(cudaDeviceSynchronize());
        for (uint32_t r = 0; r < reps; ++r)
            for (int lm = 0; lm < 2; ++lm) { // alternate the layouts, so that both see the same clocks
                CK(cudaEventRecord(e0));
                launch(lm);
                CK(cudaEventRecord(e1));
                CK(cudaEventSynchronize(e1));
                float ms = 0;
                CK(cudaEventElapsedTime(&ms, e0, e1));
                t[lm].push_back(ms);
            }
        CK(cudaGetLastError());
        for (int lm = 0; lm < 2; ++lm) {
            printf("%s %s %.1f %u", lm ? "line_major" : "chunk_major", first16 ? "offset16" : "aligned128",
                   (double)ws_lines * pitch / 1e6, reps);
            for (float x : t[lm])
                printf(" %.5f", x);
            printf("\n");
        }
    }
    CK(cudaFree(d));
    CK(cudaFree(out));
    return 0;
}
