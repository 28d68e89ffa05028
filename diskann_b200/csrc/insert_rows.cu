// insert_rows.cu — set_element for the ids of a dab_insert call (build_kernels.cu): the inmem providers write a new
// point's aux store first, then its base store (diskann-providers/.../async_/inmem/provider.rs:695-725).  Here the
// caller's rows go to a contiguous staging block at the index row stride, the encoders of every store that holds rows run
// on that block exactly as the encode-all calls run on the index rows (so the codes are byte-identical to theirs), and one
// scatter kernel then writes every record to its id: the row, the PQ codes, the SQ codes and compensation, the MinMax
// codes and compensations.  The encoders' checks (PQ: a row infinitely far from every centre; MinMax: a NaN after the
// transform) all run before anything is written, so a call that fails them leaves the index as it was.
#include "dab_common.cuh"

#include <algorithm>
#include <string>
#include <vector>

namespace dab {

namespace {

constexpr int kMaxSegments = 6;

// one fixed-size field of a record: record r is read at src + r * src_stride and written at dst + ids[r] * dst_stride
struct ScatterSegment {
    const uint8_t* src;
    uint8_t* dst;
    uint32_t src_stride, dst_stride, bytes;
};

struct ScatterParams {
    ScatterSegment seg[kMaxSegments];
    int n_segments;
    const uint32_t* ids;
    uint64_t n;
};

// One warp per record, every field of it; 16-byte (else 4-byte) accesses where both ends and the length allow them
__global__ void __launch_bounds__(256) scatter_records_kernel(const ScatterParams p) {
    const int lane = threadIdx.x & 31;
    const uint64_t warps = ((uint64_t)gridDim.x * blockDim.x) >> 5;
    for (uint64_t r = (blockIdx.x * (uint64_t)blockDim.x + threadIdx.x) >> 5; r < p.n; r += warps) {
        const uint64_t id = p.ids[r];
        for (int s = 0; s < p.n_segments; ++s) {
            const ScatterSegment g = p.seg[s];
            const uint8_t* src = g.src + r * g.src_stride;
            uint8_t* dst = g.dst + id * g.dst_stride;
            const uintptr_t align = (uintptr_t)src | (uintptr_t)dst | g.bytes;
            if (align % 16 == 0) {
                for (uint32_t i = lane; i < g.bytes / 16; i += 32) reinterpret_cast<uint4*>(dst)[i] = reinterpret_cast<const uint4*>(src)[i];
            } else if (align % 4 == 0) {
                for (uint32_t i = lane; i < g.bytes / 4; i += 32) reinterpret_cast<uint32_t*>(dst)[i] = reinterpret_cast<const uint32_t*>(src)[i];
            } else {
                for (uint32_t i = lane; i < g.bytes; i += 32) dst[i] = src[i];
            }
        }
    }
}

// the staging block of a slab of `rows` records: carved in this order, each part 256 B aligned
struct Staging {
    uint8_t* vectors = nullptr;  // [rows][row_stride], padding zeroed
    uint32_t* ids = nullptr;     // [rows]
    float* pq_f32 = nullptr;     // [rows][dim]: the rows as f32, the PQ encoder's input
    uint8_t* pq_codes = nullptr; // [rows][pq_chunks]
    uint8_t* sq_codes = nullptr; // [rows][sq.stride]
    float* sq_meta = nullptr;    // [rows][1]
    uint8_t* mm_work = nullptr;  // minmax_encode_bytes(rows)
    uint8_t* mm_codes = nullptr; // [rows][mm.stride]
    float* mm_meta = nullptr;    // [rows][4]
};

struct Stores {
    bool pq, sq, mm;  // the stores that hold rows, and so take the new ones
};

// bytes of the staging block of `rows` records; with `base` set, carves it into *s
size_t staging(const dab_index* idx, Stores st, uint64_t rows, uint8_t* base, Staging* s) {
    size_t off = 0;
    auto take = [&](size_t bytes) {
        uint8_t* p = base ? base + off : nullptr;
        off += round_up(bytes, 256);
        return p;
    };
    Staging t;
    t.vectors = take(rows * idx->row_stride);
    t.ids = (uint32_t*)take(rows * 4);
    if (st.pq) {
        t.pq_f32 = (float*)take(rows * idx->dim * 4);
        t.pq_codes = take(rows * idx->pq_chunks);
    }
    if (st.sq) {
        t.sq_codes = take(rows * idx->sq.stride);
        t.sq_meta = (float*)take(rows * idx->sq.meta_words * 4);
    }
    if (st.mm) {
        t.mm_work = take(minmax_encode_bytes(idx, rows));
        t.mm_codes = take(rows * idx->mm.stride);
        t.mm_meta = (float*)take(rows * idx->mm.meta_words * 4);
    }
    if (s) *s = t;
    return off;
}

}  // namespace

int insert_check_ids(const dab_index* idx, const uint32_t* ids, uint64_t n, const char* who) {
    if (n == 0) return DAB_OK;
    std::vector<uint32_t> seen((idx->n_points + 31) / 32, 0u);
    for (uint64_t i = 0; i < n; ++i) {
        const uint32_t id = ids[i];
        if (id >= idx->n_points)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u is not a data point (n_points %llu; start points cannot be inserted)", who, id,
                        (unsigned long long)idx->n_points);
        if (seen[id >> 5] >> (id & 31) & 1u) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u appears more than once", who, id);
        seen[id >> 5] |= 1u << (id & 31);
        if (idx->h_deleted && (idx->h_deleted[id >> 5] >> (id & 31) & 1u))
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: id %u is deleted (dab_release it first)", who, id);
    }
    return DAB_OK;
}

int insert_rows(dab_index* idx, const uint32_t* ids, const void* rows, uint64_t n, const char* who) {
    const Stores st{idx->pq_codes_ready, idx->sq.ready, idx->mm.ready};
    cudaStream_t stream = idx->stream;
    const size_t row_bytes = (size_t)idx->dim * elem_size(idx->dtype);
    // slabs of at most 256 MB of staging, as the encode-all calls use
    const size_t per_row = std::max<size_t>(1, staging(idx, st, 1, nullptr, nullptr));
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(n, (256ull << 20) / per_row));
    int rc;
    if ((rc = idx->s_stage.reserve(staging(idx, st, slab, nullptr, nullptr)))) return rc;
    Staging s;
    staging(idx, st, slab, (uint8_t*)idx->s_stage.p, &s);
    // the encoders over the slab [first, first + cnt) of the caller's rows; fails naming the caller's row
    auto encode = [&](uint64_t first, uint64_t cnt, bool write) -> int {
        DAB_CUDA(cudaMemsetAsync(s.vectors, 0, cnt * idx->row_stride, stream));
        DAB_CUDA(cudaMemcpy2DAsync(s.vectors, idx->row_stride, (const uint8_t*)rows + first * row_bytes, row_bytes, row_bytes, cnt,
                                   cudaMemcpyHostToDevice, stream));
        int rc2;
        if (st.pq) {  // dab_pq_encode_all: as_f32, then BasicTable::compress_into
            if ((rc2 = widen_rows(idx, stream, s.vectors, idx->row_stride, cnt, s.pq_f32))) return rc2;
            if ((rc2 = pq_encode_device(idx, s.pq_f32, cnt, s.pq_codes, first))) {
                std::string msg = error_buffer();
                return fail(rc2, "%s: %s", who, msg.c_str());
            }
        }
        if (st.sq && write && (rc2 = sq_encode_rows(idx, stream, s.vectors, idx->row_stride, cnt, s.sq_codes, s.sq_meta))) return rc2;
        if (st.mm) {
            unsigned long long first_nan = ~0ull;
            if ((rc2 = minmax_encode_rows(idx, stream, s.mm_work, s.vectors, idx->row_stride, cnt, s.mm_codes, s.mm_meta, &first_nan))) return rc2;
            DAB_CUDA(cudaStreamSynchronize(stream));
            if (first_nan != ~0ull)
                return fail(DAB_ERR_INVALID_ARGUMENT, "%s: row %llu contains NaN after the transform (InputContainsNaN)", who,
                            (unsigned long long)(first + first_nan));
        }
        return DAB_OK;
    };
    // more than one slab: every check first, so that a failing row leaves everything as it was
    if (slab < n)
        for (uint64_t first = 0; first < n; first += slab)
            if ((rc = encode(first, std::min(slab, n - first), false))) return rc;
    for (uint64_t first = 0; first < n; first += slab) {
        const uint64_t cnt = std::min(slab, n - first);
        if ((rc = encode(first, cnt, true))) return rc;
        DAB_CUDA(cudaMemcpyAsync(s.ids, ids + first, cnt * 4, cudaMemcpyHostToDevice, stream));
        ScatterParams p;
        memset(&p, 0, sizeof(p));
        auto add = [&](const void* src, void* dst, size_t bytes) {
            p.seg[p.n_segments++] = ScatterSegment{(const uint8_t*)src, (uint8_t*)dst, (uint32_t)bytes, (uint32_t)bytes, (uint32_t)bytes};
        };
        add(s.vectors, idx->d_vectors, idx->row_stride);
        if (st.pq) add(s.pq_codes, idx->d_codes, idx->pq_chunks);
        if (st.sq) {
            add(s.sq_codes, idx->sq.d_codes, idx->sq.stride);
            add(s.sq_meta, idx->sq.d_meta, (size_t)idx->sq.meta_words * 4);
        }
        if (st.mm) {
            add(s.mm_codes, idx->mm.d_codes, idx->mm.stride);
            add(s.mm_meta, idx->mm.d_meta, (size_t)idx->mm.meta_words * 4);
        }
        p.ids = s.ids;
        p.n = cnt;
        const int grid = (int)std::max<uint64_t>(1, std::min<uint64_t>((cnt + 7) / 8, (uint64_t)idx->sm_count * 16));
        scatter_records_kernel<<<grid, 256, 0, stream>>>(p);
        DAB_LAUNCHED();
        DAB_CUDA(cudaGetLastError());
    }
    DAB_CUDA(cudaStreamSynchronize(stream));
    ++idx->vectors_version;  // the tensor-core scan's operand copy is rebuilt on its next use
    if (st.pq) ++idx->store_writes[STORE_PQ];
    if (st.sq) ++idx->store_writes[STORE_SQ];
    if (st.mm) ++idx->store_writes[STORE_MINMAX];
    return DAB_OK;
}

}  // namespace dab
