// minmax_index.cu — the MinMax store of an index: MinMaxElement<NBITS> as the VectorRepr of an index
// (diskann-providers/src/common/minmax_repr.rs:167-336), the way diskann-garnet runs it as its traversal store
// (quantization.rs:229-362, provider.rs:1170-1358): one compressed row per point, behind an optional Hadamard transform,
// so that dab_search_batch_minmax (search_kernel_pq.cu, MODE 2) can traverse over them.
//
// Host-facing rows use the canonical-front layout of Data<NBITS> (meta/vector.rs:377-392): MinMaxCompensation {dim u32,
// b, n, a, norm_squared} (20 bytes) then ceil(dim * NBITS / 8) bytes of dense codes, value i at bit i * NBITS: a
// CodeStore with the dim word and four f32 (code_store.cu holds the rows; dim is the store's, checked on upload).  Rows
// and queries are compressed by the same launches as the standalone entry points (hadamard_transform_kernel,
// minmax_compress_kernel) into canonical rows, which the store's split brings into the device layout.
#include "dab_common.cuh"
#include "minmax.cuh"
#include "search_pq.cuh"
#include "transform.cuh"

#include <algorithm>
#include <new>

namespace dab {

namespace {

// as_f32 -> transform -> compress_into for n rows (src_stride bytes apart) into canonical rows [n][mm.row_bytes] in
// `canon`; *first_nan (device) takes the first row whose transformed vector holds a NaN.  `work` holds the f32 rows:
// n * (dim + out_dim) floats.  Queued on `stream`.
int compress_rows(const dab_index* idx, cudaStream_t stream, const void* src, size_t src_stride, uint64_t n, float* work, uint8_t* canon,
                  unsigned long long* first_nan) {
    int rc;
    if ((rc = widen_rows(idx, stream, src, src_stride, n, work))) return rc;
    const float* vec = work;
    if (idx->mm_transform) {
        float* out = work + n * idx->dim;
        DAB_CUDA(transform_launch(idx->mm_transform, idx->d_mm_tables, work, n, out, nullptr, stream));
        vec = out;
    }
    MinMaxCompressParams p;
    int warps;
    size_t smem;
    mm_compress_setup(idx->mm_grid_scale, idx->mm.dim, idx->mm.nbits, n, p, warps, smem);  // fits: checked by dab_upload_minmax
    p.vectors = vec;
    p.rows = canon;
    p.first_nan = first_nan;
    DAB_CUDA(mm_compress_launch(p, warps, smem, stream));
    return DAB_OK;
}

// the staging buffer of `n` rows through compress_rows and the split: f32 rows, canonical rows, the NaN flag
struct Staging {
    float* work;
    uint8_t* canon;
    unsigned long long* flag;
};

size_t staging_canon_off(const dab_index* idx, uint64_t n) { return round_up(n * (idx->dim + (idx->mm_transform ? idx->mm.dim : 0)) * 4, 256); }
size_t staging_flag_off(const dab_index* idx, uint64_t n) { return staging_canon_off(idx, n) + round_up(n * idx->mm.row_bytes, 256); }
size_t staging_bytes(const dab_index* idx, uint64_t n) { return staging_flag_off(idx, n) + 256; }

Staging staging_layout(const dab_index* idx, uint64_t n, uint8_t* base) {
    return Staging{(float*)base, base + staging_canon_off(idx, n), (unsigned long long*)(base + staging_flag_off(idx, n))};
}

}  // namespace

size_t minmax_encode_bytes(const dab_index* idx, uint64_t n) { return staging_bytes(idx, n); }

int minmax_encode_rows(const dab_index* idx, cudaStream_t stream, uint8_t* work, const void* src, size_t src_stride, uint64_t n, uint8_t* codes,
                       float* meta, unsigned long long* h_first_nan) {
    const Staging s = staging_layout(idx, n, work);
    int rc;
    DAB_CUDA(cudaMemsetAsync(s.flag, 0xFF, 8, stream));
    if ((rc = compress_rows(idx, stream, src, src_stride, n, s.work, s.canon, s.flag))) return rc;
    if ((rc = store_split(idx, stream, idx->mm, s.canon, n, codes, meta, nullptr))) return rc;
    DAB_CUDA(cudaMemcpyAsync(h_first_nan, s.flag, 8, cudaMemcpyDeviceToHost, stream));
    return DAB_OK;
}

void minmax_release(dab_index* idx) {
    cudaFree(idx->d_mm_tables);
    delete idx->mm_transform;
    idx->d_mm_tables = nullptr;
    idx->mm_transform = nullptr;
}

size_t minmax_stage_bytes(const dab_index* idx, uint32_t nq) { return stage_query_bytes(idx->mm, nq, staging_bytes(idx, nq)); }

int minmax_stage_queries(const dab_index* idx, cudaStream_t stream, Scratch& stage, const void* d_queries, uint32_t nq,
                         unsigned long long* h_first_nan, const uint8_t** d_qcodes, const float4** d_qmeta) {
    int rc;
    uint8_t* qcodes;
    float4* qmeta;
    if ((rc = stage_query_buffers(idx->mm, stage, nq, staging_bytes(idx, nq), &qcodes, &qmeta))) return rc;
    const Staging s = staging_layout(idx, nq, (uint8_t*)stage.p);
    DAB_CUDA(cudaMemsetAsync(s.flag, 0xFF, 8, stream));
    if ((rc = compress_rows(idx, stream, d_queries, (size_t)idx->dim * elem_size(idx->dtype), nq, s.work, s.canon, s.flag))) return rc;
    if ((rc = store_split(idx, stream, idx->mm, s.canon, nq, qcodes, (float*)qmeta, nullptr))) return rc;
    DAB_CUDA(cudaMemcpyAsync(h_first_nan, s.flag, 8, cudaMemcpyDeviceToHost, stream));
    *d_qcodes = qcodes;
    *d_qmeta = qmeta;
    return DAB_OK;
}

}  // namespace dab

using namespace dab;

static bool mm_width_ok(int nbits) { return nbits == 1 || nbits == 2 || nbits == 4 || nbits == 8; }

extern "C" {

int dab_upload_minmax(dab_index* idx, int nbits, float grid_scale, const dab_transform* t, const uint8_t* rows) {
    static const char* who = "dab_upload_minmax";
    if (!idx) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: idx is NULL", who);
    if (!mm_width_ok(nbits)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: nbits must be 1, 2, 4 or 8", who);
    if (!(grid_scale > 0.0f)) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: grid_scale must be positive (num::Positive)", who);
    if (t && t->input_dim != idx->dim)
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: the transform takes vectors of %u values, the index has %u", who, t->input_dim, idx->dim);
    const uint32_t out_dim = t ? t->output_dim : idx->dim;
    MinMaxCompressParams probe;
    int warps;
    size_t smem;
    if (!mm_compress_setup(grid_scale, out_dim, nbits, 1, probe, warps, smem))
        return fail(DAB_ERR_INVALID_ARGUMENT, "%s: rows of %u bytes do not fit the compressor's staging buffers", who, probe.row_bytes);
    DAB_CUDA(cudaSetDevice(idx->device));
    DAB_CUDA(cudaStreamSynchronize(idx->stream));
    int rc;
    if ((rc = retire_quantized_stores(idx))) return rc;  // batches in flight read the store and its transform
    ++idx->store_writes[STORE_MINMAX];
    minmax_release(idx);
    store_release(idx->mm);
    idx->mm_grid_scale = grid_scale;
    if (t) {
        idx->mm_transform = new (std::nothrow) dab_transform(*t);
        if (!idx->mm_transform) return fail(DAB_ERR_OUT_OF_MEMORY, "%s: out of host memory", who);
        const std::vector<uint32_t> tables = transform_tables(t);
        DAB_CUDA(cudaMalloc(&idx->d_mm_tables, tables.size() * 4));
        DAB_CUDA(cudaMemcpyAsync(idx->d_mm_tables, tables.data(), tables.size() * 4, cudaMemcpyHostToDevice, idx->stream));  // see store_alloc
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
    }
    if ((rc = store_alloc(idx, idx->mm, nbits, out_dim, true, 4))) return rc;  // the header: dim, then {b, n, a, norm_squared}
    return rows ? store_upload(idx, idx->mm, rows, who) : DAB_OK;
}

int dab_minmax_encode_all(dab_index* idx) {
    static const char* who = "dab_minmax_encode_all";
    int rc;
    if ((rc = store_require(idx, &dab_index::mm, "dab_upload_minmax", who))) return rc;
    if (!idx->vectors_ready) return fail(DAB_ERR_NOT_READY, "%s: vectors not uploaded", who);
    DAB_CUDA(cudaSetDevice(idx->device));
    CodeStore& mm = idx->mm;
    ++idx->store_writes[STORE_MINMAX];
    mm.ready = false;
    const uint64_t total = idx->n_total();
    const uint64_t per_row = (uint64_t)(idx->dim + (idx->mm_transform ? mm.dim : 0)) * 4 + mm.row_bytes;
    const uint64_t slab = std::max<uint64_t>(1, std::min<uint64_t>(total, (256ull << 20) / per_row));
    if ((rc = idx->s_stage.reserve(staging_bytes(idx, slab)))) return rc;
    for (uint64_t first = 0; first < total; first += slab) {
        const uint64_t cnt = std::min(slab, total - first);
        unsigned long long first_nan = ~0ull;
        if ((rc = minmax_encode_rows(idx, idx->stream, (uint8_t*)idx->s_stage.p, idx->d_vectors + first * idx->row_stride, idx->row_stride, cnt,
                                     mm.d_codes + first * mm.stride, mm.d_meta + first * mm.meta_words, &first_nan)))
            return rc;
        DAB_CUDA(cudaStreamSynchronize(idx->stream));
        if (first_nan != ~0ull)
            return fail(DAB_ERR_INVALID_ARGUMENT, "%s: row %llu contains NaN after the transform (InputContainsNaN)", who,
                        (unsigned long long)(first + first_nan));
    }
    mm.ready = true;
    return DAB_OK;
}

int dab_minmax_download(dab_index* idx, uint8_t* rows) {
    static const char* who = "dab_minmax_download";
    int rc;
    if ((rc = store_require(idx, &dab_index::mm, "dab_upload_minmax", who))) return rc;
    if (!rows) return fail(DAB_ERR_INVALID_ARGUMENT, "%s: rows is NULL", who);
    if (!idx->mm.ready) return fail(DAB_ERR_NOT_READY, "%s: no rows (dab_upload_minmax with rows, or dab_minmax_encode_all)", who);
    DAB_CUDA(cudaSetDevice(idx->device));
    return store_download(idx, idx->mm, rows);
}

}  // extern "C"
