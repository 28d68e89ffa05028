// tools/gather_peak.cu — what the H100 memory system delivers for RANDOM row gathers (the access
// pattern of every kernel on this path): each warp reads whole rows of `row_bytes` at random
// positions of a table much larger than the L2 with 16-byte loads, U rows in flight, and writes
// 4 bytes per row.  This is the practical ceiling for the frontier/search kernels, to be read
// next to the streaming-copy peak in MEASURED_PEAKS.json.
// build: nvcc -O3 -gencode arch=compute_90a,code=sm_90a -o build/gather_peak tools/gather_peak.cu
#include <cstdio>
#include <cstdlib>
#include <cuda_runtime.h>
#include <vector>

template <int U>
__global__ void __launch_bounds__(256) gather_kernel(const uint4* __restrict__ table, const unsigned* __restrict__ ids, size_t n_ids,
                                                    int row_u4, unsigned* __restrict__ out) {
    const int lane = threadIdx.x & 31;
    const size_t warp = (blockIdx.x * (size_t)blockDim.x + threadIdx.x) >> 5;
    const size_t nwarps = ((size_t)gridDim.x * blockDim.x) >> 5;
    for (size_t i0 = warp * U; i0 < n_ids; i0 += nwarps * U) {
        unsigned acc[U];
#pragma unroll
        for (int u = 0; u < U; ++u) acc[u] = 0;
        for (int off = lane; off < row_u4; off += 32) {
            uint4 v[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const size_t i = i0 + u < n_ids ? i0 + u : n_ids - 1;
                v[u] = __ldg(table + (size_t)ids[i] * row_u4 + off);
            }
#pragma unroll
            for (int u = 0; u < U; ++u) acc[u] += v[u].x ^ v[u].y ^ v[u].z ^ v[u].w;
        }
#pragma unroll
        for (int u = 0; u < U; ++u) {
            unsigned s = __reduce_add_sync(0xFFFFFFFFu, acc[u]);
            if (lane == 0 && i0 + u < n_ids) out[i0 + u] = s;
        }
    }
}

int main(int argc, char** argv) {
    const size_t n_rows = 1000000, n_ids = 12000000;
    int sm = 148;
    cudaDeviceGetAttribute(&sm, cudaDevAttrMultiProcessorCount, 0);
    for (int row_bytes : {128, 512, 1536}) {
        const int row_u4 = row_bytes / 16;
        uint4* table;
        unsigned *ids, *out;
        cudaMalloc(&table, n_rows * (size_t)row_bytes);
        cudaMemset(table, 1, n_rows * (size_t)row_bytes);
        std::vector<unsigned> h(n_ids);
        unsigned long long s = 88172645463325252ull;
        for (auto& x : h) {
            s ^= s << 13; s ^= s >> 7; s ^= s << 17;
            x = (unsigned)(s % n_rows);
        }
        cudaMalloc(&ids, n_ids * 4);
        cudaMalloc(&out, n_ids * 4);
        cudaMemcpy(ids, h.data(), n_ids * 4, cudaMemcpyHostToDevice);
        for (int variant = 0; variant < 2; ++variant) {
            cudaEvent_t e0, e1;
            cudaEventCreate(&e0);
            cudaEventCreate(&e1);
            const int grid = sm * 8;
            for (int rep = 0; rep < 3; ++rep) {
                if (variant == 0) gather_kernel<4><<<grid, 256>>>(table, ids, n_ids, row_u4, out);
                else gather_kernel<8><<<grid, 256>>>(table, ids, n_ids, row_u4, out);
            }
            cudaEventRecord(e0);
            for (int rep = 0; rep < 5; ++rep) {
                if (variant == 0) gather_kernel<4><<<grid, 256>>>(table, ids, n_ids, row_u4, out);
                else gather_kernel<8><<<grid, 256>>>(table, ids, n_ids, row_u4, out);
            }
            cudaEventRecord(e1);
            cudaEventSynchronize(e1);
            float ms = 0;
            cudaEventElapsedTime(&ms, e0, e1);
            ms /= 5;
            const double gb = (double)n_ids * (row_bytes + 8) / 1e9;
            printf("{\"row_bytes\": %d, \"rows_in_flight_per_warp\": %d, \"ms\": %.3f, \"GBps\": %.1f, \"error\": \"%s\"}\n", row_bytes,
                   variant == 0 ? 4 : 8, ms, gb / (ms / 1e3), cudaGetErrorString(cudaGetLastError()));
        }
        cudaFree(table);
        cudaFree(ids);
        cudaFree(out);
    }
    return 0;
}
