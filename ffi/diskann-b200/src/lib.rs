//! Safe wrapper over `diskann-b200-sys` (see INTEGRATION.md for how it plugs into the reference:
//! `GpuIndex` is the device snapshot a `layers::GpuFull<T>` mirrors into, `search_batch` is what a
//! `benchmark_core::search::Search` implementation (`GpuKNN`) calls once per query batch).
//! This image has no Rust toolchain: the crate is kept in step with the header by tools/gen_ffi.py
//! (the -sys half) and mirrors diskann_b200/index.py, which the tests drive through the same ABI.
use diskann_b200_sys as sys;
use std::os::raw::c_void;
use std::ptr;

/// `diskann_vector::distance::Metric` values (`#[repr(C)]`, metric.rs:8-20) — pass `metric as i32`.
#[repr(i32)]
#[derive(Clone, Copy, Debug, PartialEq, Eq)]
pub enum Metric {
    Cosine = 0,
    InnerProduct = 1,
    L2 = 2,
    CosineNormalized = 3,
}

/// Element types with a device path (VectorRepr implementors the reference instantiates).
pub trait Element: Copy {
    const DTYPE: i32;
}
impl Element for f32 {
    const DTYPE: i32 = 0;
}
impl Element for i8 {
    const DTYPE: i32 = 2;
}
impl Element for u8 {
    const DTYPE: i32 = 3;
}
// f16: `half::f16` with DTYPE = 1 (the crate does not depend on `half`; add the impl next to it)

#[derive(Debug)]
pub struct Error(pub String);
pub type Result<T> = std::result::Result<T, Error>;

fn check(status: i32) -> Result<()> {
    sys::check(status).map_err(Error)
}

/// Results of one batched search: row-major `[nq][k]`, padded with `u32::MAX` / `+inf`;
/// `cmps` / `hops` follow `SearchStats` (diskann/src/graph/index.rs:1990-1991).
pub struct Batch {
    pub k: usize,
    pub ids: Vec<u32>,
    pub dists: Vec<f32>,
    pub counts: Vec<u32>,
    pub cmps: Vec<u32>,
    pub hops: Vec<u32>,
}

/// `Range`'s parameters besides `starting_l` and `radius`, with the reference's defaults
#[derive(Clone, Copy, Debug)]
pub struct RangeArgs {
    pub beam_width: u32,
    pub inner_radius: Option<f32>,
    pub initial_slack: f32,
    pub range_slack: f32,
    pub max_returned: Option<u64>,
}

impl Default for RangeArgs {
    fn default() -> Self {
        RangeArgs { beam_width: 1, inner_radius: None, initial_slack: 1.0, range_slack: 1.0, max_returned: None }
    }
}

/// A range search batch: query q's results are `ids[offsets[q]..offsets[q + 1]]` with their distances
#[derive(Debug, Default)]
pub struct RangeBatch {
    pub offsets: Vec<u64>,
    pub ids: Vec<u32>,
    pub dists: Vec<f32>,
    pub cmps: Vec<u32>,
    pub hops: Vec<u32>,
    pub second_round: Vec<u8>,
}

pub struct GpuIndex<T: Element> {
    raw: *mut sys::dab_index,
    dim: usize,
    _marker: std::marker::PhantomData<T>,
}

// one CUDA stream per handle; read-only calls from one thread at a time (INTEGRATION.md §6)
unsafe impl<T: Element> Send for GpuIndex<T> {}

impl<T: Element> GpuIndex<T> {
    pub fn new(metric: Metric, dim: usize, n_points: u64, n_start: u32, max_degree: u32, device: i32) -> Result<Self> {
        let mut raw = ptr::null_mut();
        check(unsafe { sys::dab_create(&mut raw, T::DTYPE, metric as i32, dim as u32, n_points, n_start, max_degree, device) })?;
        Ok(Self { raw, dim, _marker: std::marker::PhantomData })
    }

    /// Dense row-major rows `[count][dim]` starting at row `first` (start points follow the data points).
    pub fn upload_vectors(&mut self, rows: &[T], first: u64) -> Result<()> {
        assert_eq!(rows.len() % self.dim, 0, "rows must be a whole number of vectors");
        check(unsafe { sys::dab_upload_vectors(self.raw, rows.as_ptr() as *const c_void, first, (rows.len() / self.dim) as u64) })
    }

    /// Adjacency rows `[count][stride]` with `row[0] = degree` (diskann-inmem/src/neighbors.rs:69-163).
    pub fn upload_graph(&mut self, adj: &[u32], stride: u32, first: u64) -> Result<()> {
        assert_eq!(adj.len() % stride as usize, 0);
        check(unsafe { sys::dab_upload_graph(self.raw, adj.as_ptr(), stride, first, (adj.len() / stride as usize) as u64) })
    }

    /// Batched `multi_insert`-style construction on the device over the uploaded vectors.
    pub fn build(&mut self, pruned_degree: u32, l_build: u32, alpha: f32) -> Result<()> {
        check(unsafe { sys::dab_build(self.raw, pruned_degree, l_build, alpha, 0) })
    }

    /// `DiskANNIndex::insert` / `multi_insert` into the graph as it stands: dense rows `[ids.len()][dim]` become the
    /// points `ids`, linked in consecutive chunks of `batch_size` (0: 65536).
    pub fn insert(&mut self, ids: &[u32], rows: &[T], pruned_degree: u32, l_build: u32, alpha: f32, batch_size: u32) -> Result<()> {
        assert_eq!(rows.len(), ids.len() * self.dim, "one row per id");
        check(unsafe {
            sys::dab_insert(self.raw, ids.as_ptr(), rows.as_ptr() as *const c_void, ids.len() as u64, pruned_degree, l_build, alpha,
                            batch_size)
        })
    }

    /// `Delete::delete`: every k-NN search then leaves these points out of its results.
    pub fn delete(&mut self, ids: &[u32]) -> Result<()> {
        check(unsafe { sys::dab_delete(self.raw, ids.as_ptr(), ids.len() as u64) })
    }

    /// `Delete::release`: clears the deletion mark and empties the adjacency rows of deleted points.
    pub fn release(&mut self, ids: &[u32]) -> Result<()> {
        check(unsafe { sys::dab_release(self.raw, ids.as_ptr(), ids.len() as u64) })
    }

    /// `Delete::status_by_internal_id` for each id: true when deleted.
    pub fn delete_status(&self, ids: &[u32]) -> Result<Vec<bool>> {
        let mut out = vec![0u8; ids.len()];
        check(unsafe { sys::dab_delete_status(self.raw, ids.as_ptr(), ids.len() as u64, out.as_mut_ptr()) })?;
        Ok(out.into_iter().map(|b| b != 0).collect())
    }

    /// `consolidate_vector` for every node; returns the number of lists rewritten.
    pub fn consolidate(&mut self, pruned_degree: u32, alpha: f32) -> Result<u64> {
        let mut rewritten = 0u64;
        check(unsafe { sys::dab_consolidate(self.raw, pruned_degree, alpha, &mut rewritten) })?;
        Ok(rewritten)
    }

    /// `multi_inplace_delete` in chunks of `batch_size` (1: `inplace_delete` id by id, 0: one chunk); `method` is one
    /// of the DAB_INPLACE_* values of diskann_b200.h: 0 VisitedAndTopK (with `k_value`, `l_value`), 1 TwoHopAndOneHop, 2 OneHop.
    #[allow(clippy::too_many_arguments)]
    pub fn inplace_delete(&mut self, ids: &[u32], num_to_replace: u32, method: i32, pruned_degree: u32, alpha: f32, k_value: u32,
                          l_value: u32, batch_size: u32) -> Result<()> {
        check(unsafe {
            sys::dab_inplace_delete(self.raw, ids.as_ptr(), ids.len() as u64, method, num_to_replace, k_value, l_value, pruned_degree, alpha,
                                    batch_size)
        })
    }

    /// `drop_deleted_neighbors` for every node; returns the number of lists rewritten.
    pub fn drop_deleted_neighbors(&mut self, pruned_degree: u32, only_orphans: bool) -> Result<u64> {
        let mut rewritten = 0u64;
        check(unsafe { sys::dab_drop_deleted_neighbors(self.raw, pruned_degree, only_orphans as i32, &mut rewritten) })?;
        Ok(rewritten)
    }

    /// `count_reachable_nodes` from `start_ids` (`None`: the index's start points).
    pub fn count_reachable(&self, start_ids: Option<&[u32]>) -> Result<u64> {
        let mut count = 0u64;
        let none = [0u32; 1]; // an empty list still passes a pointer: NULL means the start points
        let (ptr, n) = match start_ids {
            None => (std::ptr::null(), 0),
            Some(ids) => (if ids.is_empty() { none.as_ptr() } else { ids.as_ptr() }, ids.len() as u32),
        };
        check(unsafe { sys::dab_count_reachable(self.raw, ptr, n, &mut count) })?;
        Ok(count)
    }

    /// `get_degree_stats` over `ids` (`None`: every id): (max_degree, avg_degree, min_degree, cnt_less_than_two).
    pub fn degree_stats(&self, ids: Option<&[u32]>) -> Result<(u32, f32, u32, u64)> {
        let (mut mx, mut avg, mut mn, mut lt2) = (0u32, 0f32, 0u32, 0u64);
        let none = [0u32; 1];
        let (ptr, n) = match ids {
            None => (std::ptr::null(), 0),
            Some(ids) => (if ids.is_empty() { none.as_ptr() } else { ids.as_ptr() }, ids.len() as u64),
        };
        check(unsafe { sys::dab_degree_stats(self.raw, ptr, n, &mut mx, &mut avg, &mut mn, &mut lt2) })?;
        Ok((mx, avg, mn, lt2))
    }

    /// `prune_range` over `ids` (`None`: every id); returns the number of lists rewritten.
    pub fn prune_range(&mut self, ids: Option<&[u32]>, pruned_degree: u32, alpha: f32) -> Result<u64> {
        let mut rewritten = 0u64;
        let none = [0u32; 1];
        let (ptr, n) = match ids {
            None => (std::ptr::null(), 0),
            Some(ids) => (if ids.is_empty() { none.as_ptr() } else { ids.as_ptr() }, ids.len() as u64),
        };
        check(unsafe { sys::dab_prune_range(self.raw, ptr, n, pruned_degree, alpha, &mut rewritten) })?;
        Ok(rewritten)
    }

    /// `KNN::search` for every query of the batch at once (search_internal + post-processing).
    pub fn search_batch(&self, queries: &[T], k: usize, l_search: u32, beam_width: u32) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width,
                                  b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// The attribute of ids `first ..` for `search_batch_diverse` (the reference's `AttributeValueProvider`); `present`
    /// `None`: every id of the range has its value, else `false` marks an id without an attribute.
    pub fn upload_attributes(&mut self, values: &[u32], present: Option<&[bool]>, first: u64) -> Result<()> {
        let flags: Option<Vec<u8>> = present.map(|p| {
            assert_eq!(p.len(), values.len());
            p.iter().map(|&b| b as u8).collect()
        });
        check(unsafe {
            sys::dab_upload_attributes(self.raw, values.as_ptr(), flags.as_ref().map_or(std::ptr::null(), |f| f.as_ptr()), first,
                                       values.len() as u64)
        })
    }

    /// `Diverse::search` (diverse_search.rs:189-234): at most `diverse_k` results per attribute value.
    pub fn search_batch_diverse(&self, queries: &[T], k: usize, l_search: u32, diverse_k: u32, beam_width: u32) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_diverse(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width, diverse_k,
                                          b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(),
                                          b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// The 64-bit label sets of ids `first ..` for `search_batch_filtered`.
    pub fn upload_labels(&mut self, labels: &[u64], first: u64) -> Result<()> {
        check(unsafe { sys::dab_upload_labels(self.raw, labels.as_ptr(), first, labels.len() as u64) })
    }

    /// `InlineFilterSearch::search` (inline_filter_search.rs:89-160): query q accepts id i when `labels[i] & masks[q]` is
    /// non-zero (`match_all` false) or equals `masks[q]` (`match_all` true); `adaptive_l`: `None` or `(samples, scale)`,
    /// the reference's `AdaptiveL` (samples >= 1).
    pub fn search_batch_filtered(&self, queries: &[T], masks: &[u64], k: usize, l_search: u32, beam_width: u32, match_all: bool,
                                 adaptive_l: Option<(u32, f64)>) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        assert_eq!(masks.len(), nq);
        let (samples, scale) = adaptive_l.unwrap_or((0, 1.0));
        assert!(adaptive_l.is_none() || samples > 0, "AdaptiveL: sample count cannot be zero");
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_filtered(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width,
                                           masks.as_ptr(), match_all as u32, samples, scale, b.ids.as_mut_ptr(), b.dists.as_mut_ptr(),
                                           b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// `search_batch_filtered` with the traversal distances of `search_batch_pq` (the PQ store); `rerank`: the
    /// full-precision `Rerank` of the first L matches.
    #[allow(clippy::too_many_arguments)]
    pub fn search_batch_filtered_pq(&self, queries: &[T], masks: &[u64], k: usize, l_search: u32, beam_width: u32, match_all: bool,
                                    adaptive_l: Option<(u32, f64)>, rerank: bool) -> Result<Batch> {
        self.filtered_quantized(sys::dab_search_batch_filtered_pq, queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank)
    }

    /// `search_batch_filtered` with the traversal distances of `search_batch_sq` (the scalar-quantized store).
    #[allow(clippy::too_many_arguments)]
    pub fn search_batch_filtered_sq(&self, queries: &[T], masks: &[u64], k: usize, l_search: u32, beam_width: u32, match_all: bool,
                                    adaptive_l: Option<(u32, f64)>, rerank: bool) -> Result<Batch> {
        self.filtered_quantized(sys::dab_search_batch_filtered_sq, queries, masks, k, l_search, beam_width, match_all, adaptive_l, rerank)
    }

    /// `search_batch_filtered` with the traversal distances of `search_batch_minmax` (the MinMax store).
    #[allow(clippy::too_many_arguments)]
    pub fn search_batch_filtered_minmax(&self, queries: &[T], masks: &[u64], k: usize, l_search: u32, beam_width: u32, match_all: bool,
                                        adaptive_l: Option<(u32, f64)>, rerank: bool) -> Result<Batch> {
        self.filtered_quantized(sys::dab_search_batch_filtered_minmax, queries, masks, k, l_search, beam_width, match_all, adaptive_l,
                                rerank)
    }

    #[allow(clippy::too_many_arguments)]
    fn filtered_quantized(&self, f: FilteredQuantized, queries: &[T], masks: &[u64], k: usize, l_search: u32, beam_width: u32,
                          match_all: bool, adaptive_l: Option<(u32, f64)>, rerank: bool) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        assert_eq!(masks.len(), nq);
        let (samples, scale) = adaptive_l.unwrap_or((0, 1.0));
        assert!(adaptive_l.is_none() || samples > 0, "AdaptiveL: sample count cannot be zero");
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            f(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width, masks.as_ptr(), match_all as u32, samples,
              scale, rerank as i32, b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// `Range::search` (range_search.rs:255-469) for the batch: every point within `radius` of each query, query q's
    /// results at `offsets[q] .. offsets[q + 1]` in the reference's output order.
    pub fn range_search(&self, queries: &[T], l_search: u32, radius: f32, args: RangeArgs) -> Result<RangeBatch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut set: *mut sys::dab_range = std::ptr::null_mut();
        check(unsafe {
            sys::dab_range_search(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, args.beam_width, radius,
                                  args.inner_radius.is_some() as i32, args.inner_radius.unwrap_or(0.0), args.initial_slack,
                                  args.range_slack, args.max_returned.unwrap_or(0), &mut set)
        })?;
        take_range(set, nq)
    }

    /// `FilteredRange::search` (filtered_range_search.rs:119-248) for the batch: every point within `radius` of each
    /// query that its mask accepts (`masks`: one per query; `match_all`: ALL, else ANY, as `search_batch_filtered`).
    pub fn range_search_filtered(&self, queries: &[T], masks: &[u64], match_all: bool, l_search: u32, radius: f32, args: RangeArgs)
        -> Result<RangeBatch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        assert_eq!(masks.len(), nq);
        let mut set: *mut sys::dab_range = std::ptr::null_mut();
        check(unsafe {
            sys::dab_range_search_filtered(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, args.beam_width, radius,
                                           args.inner_radius.is_some() as i32, args.inner_radius.unwrap_or(0.0), args.initial_slack,
                                           args.range_slack, args.max_returned.unwrap_or(0), masks.as_ptr(), match_all as u32, &mut set)
        })?;
        take_range(set, nq)
    }

    /// `range_search` with every distance of both phases the PQ store's (those of `search_batch_pq`); `rerank`: the
    /// in_range ids by full-precision distance, those within (inner_radius, radius] of it, sorted by it, with it.
    pub fn range_search_pq(&self, queries: &[T], l_search: u32, radius: f32, args: RangeArgs, rerank: bool) -> Result<RangeBatch> {
        self.range_quantized(sys::dab_range_search_pq, queries, l_search, radius, args, rerank)
    }

    /// `range_search_pq` over the scalar-quantized store (the distances of `search_batch_sq`).
    pub fn range_search_sq(&self, queries: &[T], l_search: u32, radius: f32, args: RangeArgs, rerank: bool) -> Result<RangeBatch> {
        self.range_quantized(sys::dab_range_search_sq, queries, l_search, radius, args, rerank)
    }

    /// `range_search_pq` over the MinMax store (the distances of `search_batch_minmax`).
    pub fn range_search_minmax(&self, queries: &[T], l_search: u32, radius: f32, args: RangeArgs, rerank: bool) -> Result<RangeBatch> {
        self.range_quantized(sys::dab_range_search_minmax, queries, l_search, radius, args, rerank)
    }

    /// `range_search_filtered` with every distance of both phases the PQ store's (those of `search_batch_pq`); `rerank`:
    /// the returned matches by full-precision distance, sorted by it (NaN last), those above inner_radius, with it (no
    /// outer-radius filter, as in `FilteredRange::search`).
    pub fn range_search_filtered_pq(&self, queries: &[T], masks: &[u64], match_all: bool, l_search: u32, radius: f32, args: RangeArgs,
                                    rerank: bool) -> Result<RangeBatch> {
        self.range_filtered_quantized(sys::dab_range_search_filtered_pq, queries, masks, match_all, l_search, radius, args, rerank)
    }

    /// `range_search_filtered_pq` over the scalar-quantized store (the distances of `search_batch_sq`).
    pub fn range_search_filtered_sq(&self, queries: &[T], masks: &[u64], match_all: bool, l_search: u32, radius: f32, args: RangeArgs,
                                    rerank: bool) -> Result<RangeBatch> {
        self.range_filtered_quantized(sys::dab_range_search_filtered_sq, queries, masks, match_all, l_search, radius, args, rerank)
    }

    /// `range_search_filtered_pq` over the MinMax store (the distances of `search_batch_minmax`).
    pub fn range_search_filtered_minmax(&self, queries: &[T], masks: &[u64], match_all: bool, l_search: u32, radius: f32, args: RangeArgs,
                                        rerank: bool) -> Result<RangeBatch> {
        self.range_filtered_quantized(sys::dab_range_search_filtered_minmax, queries, masks, match_all, l_search, radius, args, rerank)
    }

    #[allow(clippy::too_many_arguments)]
    fn range_filtered_quantized(&self, f: RangeFilteredQuantized, queries: &[T], masks: &[u64], match_all: bool, l_search: u32, radius: f32,
                                args: RangeArgs, rerank: bool) -> Result<RangeBatch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        assert_eq!(masks.len(), nq);
        let mut set: *mut sys::dab_range = std::ptr::null_mut();
        check(unsafe {
            f(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, args.beam_width, radius, args.inner_radius.is_some() as i32,
              args.inner_radius.unwrap_or(0.0), args.initial_slack, args.range_slack, args.max_returned.unwrap_or(0), masks.as_ptr(),
              match_all as u32, rerank as i32, &mut set)
        })?;
        take_range(set, nq)
    }

    fn range_quantized(&self, f: RangeQuantized, queries: &[T], l_search: u32, radius: f32, args: RangeArgs, rerank: bool)
        -> Result<RangeBatch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut set: *mut sys::dab_range = std::ptr::null_mut();
        check(unsafe {
            f(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, args.beam_width, radius, args.inner_radius.is_some() as i32,
              args.inner_radius.unwrap_or(0.0), args.initial_slack, args.range_slack, args.max_returned.unwrap_or(0), rerank as i32, &mut set)
        })?;
        take_range(set, nq)
    }

    /// `search_batch_diverse` with the traversal distances of `search_batch_pq` (the PQ store); `rerank`: the
    /// full-precision `Rerank` of the post-processed list.
    pub fn search_batch_diverse_pq(&self, queries: &[T], k: usize, l_search: u32, diverse_k: u32, beam_width: u32, rerank: bool) -> Result<Batch> {
        self.diverse_quantized(sys::dab_search_batch_diverse_pq, queries, k, l_search, diverse_k, beam_width, rerank)
    }

    /// `search_batch_diverse` with the traversal distances of `search_batch_sq` (the scalar-quantized store).
    pub fn search_batch_diverse_sq(&self, queries: &[T], k: usize, l_search: u32, diverse_k: u32, beam_width: u32, rerank: bool) -> Result<Batch> {
        self.diverse_quantized(sys::dab_search_batch_diverse_sq, queries, k, l_search, diverse_k, beam_width, rerank)
    }

    /// `search_batch_diverse` with the traversal distances of `search_batch_minmax` (the MinMax store).
    pub fn search_batch_diverse_minmax(&self, queries: &[T], k: usize, l_search: u32, diverse_k: u32, beam_width: u32, rerank: bool)
        -> Result<Batch> {
        self.diverse_quantized(sys::dab_search_batch_diverse_minmax, queries, k, l_search, diverse_k, beam_width, rerank)
    }

    #[allow(clippy::too_many_arguments)]
    fn diverse_quantized(&self, f: DiverseQuantized, queries: &[T], k: usize, l_search: u32, diverse_k: u32, beam_width: u32, rerank: bool)
        -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            f(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width, diverse_k, rerank as i32,
              b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// Queue a batch on `slot` without waiting (`search_all`'s one task per partition, api.rs:410-419, mapped to
    /// device slots).  The returned guard borrows the queries and owns the result buffers; `InFlight::wait` joins it.
    pub fn search_batch_async<'a>(&'a self, slot: u32, queries: &'a [T], k: usize, l_search: u32, beam_width: u32) -> Result<InFlight<'a, T>> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_async(self.raw, slot, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width,
                                        b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(InFlight { index: self, slot, batch: Some(b), _queries: queries })
    }

    /// PQ traversal + the providers' full-precision `Rerank` (what `use_fp_for_search: false` runs).
    pub fn search_batch_pq_rerank(&self, queries: &[T], k: usize, l_search: u32, beam_width: u32) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_pq_rerank(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width,
                                            b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(),
                                            b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// `train_pq` + encoding of every stored row, on the device.
    pub fn train_pq(&mut self, train: &[f32], n_chunks: u32, seed: u64) -> Result<()> {
        assert_eq!(train.len() % self.dim, 0);
        check(unsafe { sys::dab_pq_train(self.raw, train.as_ptr(), (train.len() / self.dim) as u64, n_chunks, 256, 5, seed) })?;
        check(unsafe { sys::dab_pq_encode_all(self.raw) })
    }

    /// The scalar-quantized store (`SQStore<NBITS>`): hand over the quantizer, encode every resident row on the device.
    pub fn set_scalar_quantizer(&mut self, nbits: i32, shift: &[f32], scale: f32, shift_square_norm: f32, mean_norm: Option<f32>) -> Result<()> {
        assert_eq!(shift.len(), self.dim);
        check(unsafe {
            sys::dab_upload_sq(self.raw, nbits, shift.as_ptr(), scale, shift_square_norm, mean_norm.unwrap_or(0.0), std::ptr::null())
        })?;
        check(unsafe { sys::dab_sq_encode_all(self.raw) })
    }

    /// Traversal over the scalar-quantized rows; `rerank` adds `Pipeline<FilterStartPoints, Rerank>`.
    pub fn search_batch_sq(&self, queries: &[T], k: usize, l_search: u32, beam_width: u32, rerank: bool) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_sq(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width, rerank as i32,
                                     b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(),
                                     b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// The MinMax store (`MinMaxElement<NBITS>` as the vector representation): `MinMaxQuantizer::new(transform, or
    /// Transform::Null, grid_scale)`, every resident row encoded on the device.  The index keeps its own copy of the
    /// transform.
    pub fn set_minmax_quantizer(&mut self, nbits: i32, grid_scale: f32, transform: Option<&Transform>) -> Result<()> {
        let t = transform.map_or(std::ptr::null(), |t| t.raw as *const sys::dab_transform);
        check(unsafe { sys::dab_upload_minmax(self.raw, nbits, grid_scale, t, std::ptr::null()) })?;
        check(unsafe { sys::dab_minmax_encode_all(self.raw) })
    }

    /// Traversal over the MinMax rows (queries compressed by the store's quantizer); `rerank` adds
    /// `Pipeline<FilterStartPoints, Rerank>`.
    pub fn search_batch_minmax(&self, queries: &[T], k: usize, l_search: u32, beam_width: u32, rerank: bool) -> Result<Batch> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_search_batch_minmax(self.raw, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width,
                                         rerank as i32, b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(),
                                         b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }

    /// `search_batch_pq_rerank` (`rerank`) or the PQ traversal alone, queued on `slot` without waiting: the quantized
    /// counterpart of `search_batch_async`, with bit-identical results.  Slots are shared by batches of every kind.
    pub fn search_batch_pq_async<'a>(&'a self, slot: u32, queries: &'a [T], k: usize, l_search: u32, beam_width: u32, rerank: bool)
        -> Result<InFlight<'a, T>> {
        self.quantized_async(sys::dab_search_batch_pq_async, slot, queries, k, l_search, beam_width, rerank)
    }

    /// `search_batch_sq` queued on `slot` without waiting.
    pub fn search_batch_sq_async<'a>(&'a self, slot: u32, queries: &'a [T], k: usize, l_search: u32, beam_width: u32, rerank: bool)
        -> Result<InFlight<'a, T>> {
        self.quantized_async(sys::dab_search_batch_sq_async, slot, queries, k, l_search, beam_width, rerank)
    }

    /// `search_batch_minmax` queued on `slot` without waiting.  A query holding a NaN after the transform makes
    /// `InFlight::wait` fail with the synchronous call's error.
    pub fn search_batch_minmax_async<'a>(&'a self, slot: u32, queries: &'a [T], k: usize, l_search: u32, beam_width: u32, rerank: bool)
        -> Result<InFlight<'a, T>> {
        self.quantized_async(sys::dab_search_batch_minmax_async, slot, queries, k, l_search, beam_width, rerank)
    }

    #[allow(clippy::too_many_arguments)]
    fn quantized_async<'a>(&'a self, launch: QuantizedAsync, slot: u32, queries: &'a [T], k: usize, l_search: u32, beam_width: u32,
                           rerank: bool) -> Result<InFlight<'a, T>> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            launch(self.raw, slot, queries.as_ptr() as *const c_void, nq as u32, k as u32, l_search, beam_width, rerank as i32,
                   b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(), b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(InFlight { index: self, slot, batch: Some(b), _queries: queries })
    }

    /// `DiskANNIndex::paged_search` for every query of the batch: each `PagedSearch::next_page(k)` resumes the
    /// queries' searches on the device and returns their next pages (graph/search/paged.rs:53-149).
    pub fn paged_search(&self, queries: &[T], l_search: u32) -> Result<PagedSearch<'_, T>> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut raw = ptr::null_mut();
        check(unsafe { sys::dab_paged_search_begin(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, &mut raw) })?;
        Ok(PagedSearch { raw, nq, _index: self })
    }

    /// `paged_search` with the PQ traversal distances (TableL2 / TableIP, DirectCosine for `Metric::Cosine`); pages
    /// return them (the reference's paged search has no post-processing, so no rerank).
    pub fn paged_search_pq(&self, queries: &[T], l_search: u32) -> Result<PagedSearch<'_, T>> {
        self.paged_search_with(sys::dab_paged_search_begin_pq, queries, l_search)
    }

    /// `paged_search` through the scalar-quantized store; no rerank.
    pub fn paged_search_sq(&self, queries: &[T], l_search: u32) -> Result<PagedSearch<'_, T>> {
        self.paged_search_with(sys::dab_paged_search_begin_sq, queries, l_search)
    }

    /// `paged_search` through the MinMax store; no rerank.  A query holding a NaN after the transform is an error.
    pub fn paged_search_minmax(&self, queries: &[T], l_search: u32) -> Result<PagedSearch<'_, T>> {
        self.paged_search_with(sys::dab_paged_search_begin_minmax, queries, l_search)
    }

    fn paged_search_with(&self, begin: PagedBegin, queries: &[T], l_search: u32) -> Result<PagedSearch<'_, T>> {
        assert_eq!(queries.len() % self.dim, 0);
        let nq = queries.len() / self.dim;
        let mut raw = ptr::null_mut();
        check(unsafe { begin(self.raw, queries.as_ptr() as *const c_void, nq as u32, l_search, &mut raw) })?;
        Ok(PagedSearch { raw, nq, _index: self })
    }

    /// One process per GPU: join the communicator described by `id` (from `unique_id()` on rank 0) …
    pub fn comm_init(&mut self, id: &[u8; 128], n_ranks: i32, rank: i32) -> Result<()> {
        check(unsafe { sys::dab_comm_init(self.raw, id.as_ptr() as *const _, n_ranks, rank) })
    }

    /// … and replicate the resident snapshot from `root` (one NCCL broadcast per buffer, at load).
    pub fn broadcast_index(&mut self, root: i32) -> Result<()> {
        check(unsafe { sys::dab_broadcast_index(self.raw, root) })
    }
}

/// The host-buffer `_async` entry points of the quantized traversals (one signature for PQ, SQ and MinMax).
type QuantizedAsync = unsafe extern "C" fn(*mut sys::dab_index, u32, *const c_void, u32, u32, u32, u32, std::os::raw::c_int, *mut u32,
                                           *mut f32, *mut u32, *mut u32, *mut u32) -> std::os::raw::c_int;

/// The entry points that open a paged search over a quantized store (one signature for PQ, SQ and MinMax).
type DiverseQuantized = unsafe extern "C" fn(*mut sys::dab_index, *const c_void, u32, u32, u32, u32, u32, std::os::raw::c_int,
                                             *mut u32, *mut f32, *mut u32, *mut u32, *mut u32) -> std::os::raw::c_int;
type FilteredQuantized = unsafe extern "C" fn(*mut sys::dab_index, *const c_void, u32, u32, u32, u32, *const u64, u32, u32, f64,
                                              std::os::raw::c_int, *mut u32, *mut f32, *mut u32, *mut u32, *mut u32) -> std::os::raw::c_int;
type RangeQuantized = unsafe extern "C" fn(*mut sys::dab_index, *const c_void, u32, u32, u32, f32, std::os::raw::c_int, f32, f32, f32, u64,
                                           std::os::raw::c_int, *mut *mut sys::dab_range) -> std::os::raw::c_int;
type RangeFilteredQuantized = unsafe extern "C" fn(*mut sys::dab_index, *const c_void, u32, u32, u32, f32, std::os::raw::c_int, f32, f32, f32,
                                                   u64, *const u64, u32, std::os::raw::c_int, *mut *mut sys::dab_range)
                                                   -> std::os::raw::c_int;

/// The offsets, stats and results of a range search's result set, which is freed
fn take_range(set: *mut sys::dab_range, nq: usize) -> Result<RangeBatch> {
    let mut r = RangeBatch { offsets: vec![0; nq + 1], ids: Vec::new(), dists: Vec::new(), cmps: vec![0; nq], hops: vec![0; nq],
                             second_round: vec![0; nq] };
    let rc = unsafe { sys::dab_range_offsets(set, r.offsets.as_mut_ptr(), r.cmps.as_mut_ptr(), r.hops.as_mut_ptr(), r.second_round.as_mut_ptr()) };
    if rc == 0 {
        let total = r.offsets[nq] as usize;
        r.ids = vec![0; total];
        r.dists = vec![0.0; total];
    }
    let rc = if rc == 0 { unsafe { sys::dab_range_results(set, r.ids.as_mut_ptr(), r.dists.as_mut_ptr()) } } else { rc };
    unsafe { sys::dab_range_free(set) };
    check(rc)?;
    Ok(r)
}

type PagedBegin = unsafe extern "C" fn(*mut sys::dab_index, *const c_void, u32, u32, *mut *mut sys::dab_paged) -> std::os::raw::c_int;

/// A batch in flight on one slot of the device.  Dropping it joins the slot (the library writes into the
/// buffers it owns until then).
pub struct InFlight<'a, T: Element> {
    index: &'a GpuIndex<T>,
    slot: u32,
    batch: Option<Batch>,
    _queries: &'a [T],
}

impl<'a, T: Element> InFlight<'a, T> {
    pub fn wait(mut self) -> Result<Batch> {
        check(unsafe { sys::dab_wait(self.index.raw, self.slot) })?;
        Ok(self.batch.take().expect("joined once"))
    }
}

impl<'a, T: Element> Drop for InFlight<'a, T> {
    fn drop(&mut self) {
        if self.batch.is_some() {
            unsafe { sys::dab_wait(self.index.raw, self.slot) };
        }
    }
}

/// A paged search over a query batch; it borrows the index, so the index outlives it and cannot be changed under it.
pub struct PagedSearch<'a, T: Element> {
    raw: *mut sys::dab_paged,
    nq: usize,
    _index: &'a GpuIndex<T>,
}

impl<'a, T: Element> PagedSearch<'a, T> {
    /// The next page of at most `k` results per query (`0 < k <= l_search`): `counts[q] == 0` once query `q` is
    /// exhausted; `cmps` / `hops` are the session's cumulative counts.
    pub fn next_page(&mut self, k: usize) -> Result<Batch> {
        let nq = self.nq;
        let mut b = Batch { k, ids: vec![0; nq * k], dists: vec![0.0; nq * k], counts: vec![0; nq], cmps: vec![0; nq], hops: vec![0; nq] };
        check(unsafe {
            sys::dab_paged_search_next(self.raw, k as u32, b.ids.as_mut_ptr(), b.dists.as_mut_ptr(), b.counts.as_mut_ptr(),
                                       b.cmps.as_mut_ptr(), b.hops.as_mut_ptr())
        })?;
        Ok(b)
    }
}

impl<'a, T: Element> Drop for PagedSearch<'a, T> {
    fn drop(&mut self) {
        unsafe { sys::dab_paged_search_end(self.raw) }
    }
}

pub fn unique_id() -> Result<[u8; 128]> {
    let mut id = [0u8; 128];
    check(unsafe { sys::dab_comm_unique_id(id.as_mut_ptr() as *mut _) })?;
    Ok(id)
}

impl<T: Element> Drop for GpuIndex<T> {
    fn drop(&mut self) {
        unsafe { sys::dab_destroy(self.raw) }
    }
}

/// `MinMaxQuantizer::new(Transform::Null(dim), grid_scale)` + `compress_into` for `vectors.len() / dim` vectors:
/// rows in the canonical-front layout of `minmax::Data<NBITS>` (`DataRef::from_canonical_front(&row, dim)`), and the
/// `L2Loss` of every vector.  `Err` when an input vector contains NaN (`InputContainsNaN`).
pub fn minmax_compress(device: i32, grid_scale: f32, dim: usize, nbits: i32, vectors: &[f32]) -> Result<(Vec<u8>, Vec<f32>)> {
    let n = vectors.len() / dim;
    let row_bytes = unsafe { sys::dab_minmax_row_bytes(dim as u32, nbits) } as usize;
    let mut rows = vec![0u8; n * row_bytes];
    let mut loss = vec![0f32; n];
    check(unsafe {
        sys::dab_minmax_compress(device, grid_scale, dim as u32, nbits, vectors.as_ptr(), n as u64, rows.as_mut_ptr(), loss.as_mut_ptr())
    })?;
    Ok((rows, loss))
}

/// `MinMax{L2Squared, IP, Cosine, CosineNormalized}::evaluate(DataRef<N>, DataRef<M>)` for row pairs (N x N or 8 x N bits).
pub fn minmax_distances(device: i32, metric: Metric, nbits_x: i32, nbits_y: i32, dim: usize, x_rows: &[u8], y_rows: &[u8]) -> Result<Vec<f32>> {
    let n = x_rows.len() / unsafe { sys::dab_minmax_row_bytes(dim as u32, nbits_x) } as usize;
    let mut out = vec![0f32; n];
    check(unsafe {
        sys::dab_minmax_distances(device, metric as i32, nbits_x, nbits_y, dim as u32, x_rows.as_ptr(), y_rows.as_ptr(), n as u64, out.as_mut_ptr())
    })?;
    Ok(out)
}

/// Full-precision queries (`FullQuery`) against compressed rows: `MinMax*::evaluate(FullQueryRef, DataRef<NBITS>)` for
/// every (query, row) pair, row-major `[nq][n]`.
pub fn minmax_query_distances(device: i32, metric: Metric, nbits: i32, dim: usize, queries: &[f32], rows: &[u8]) -> Result<Vec<f32>> {
    let nq = queries.len() / dim;
    let n = rows.len() / unsafe { sys::dab_minmax_row_bytes(dim as u32, nbits) } as usize;
    let mut out = vec![0f32; nq * n];
    check(unsafe {
        sys::dab_minmax_query_distances(device, metric as i32, nbits, dim as u32, queries.as_ptr(), nq as u32, rows.as_ptr(), n as u64, out.as_mut_ptr())
    })?;
    Ok(out)
}

/// `Transform::PaddingHadamard` / `Transform::DoubleHadamard` (diskann-quantization/src/algorithms/transforms) from the
/// parts the reference serializes (`try_from_parts`); signs are the flatbuffer's bools.  A host-side object: only
/// `apply` and the MinMax calls below touch the device.
pub struct Transform {
    raw: *mut sys::dab_transform,
}

// immutable after creation: every call takes it by const pointer
unsafe impl Send for Transform {}
unsafe impl Sync for Transform {}

impl Transform {
    fn create(kind: i32, signs0: &[bool], inner_dim: usize, signs1: Option<&[bool]>, subsample: Option<&[u32]>) -> Result<Self> {
        let s0: Vec<u8> = signs0.iter().map(|&b| b as u8).collect();
        let s1: Option<Vec<u8>> = signs1.map(|s| s.iter().map(|&b| b as u8).collect());
        let mut raw = ptr::null_mut();
        check(unsafe {
            sys::dab_transform_create(
                &mut raw,
                kind,
                s0.len() as u32,
                inner_dim as u32,
                s0.as_ptr(),
                s1.as_ref().map_or(ptr::null(), |s| s.as_ptr()),
                // `Some(&[])` must stay distinguishable from `None` (SubsampleEmpty): a dangling non-null pointer
                subsample.map_or(ptr::null(), |s| s.as_ptr()),
                subsample.map_or(0, |s| s.len() as u32),
            )
        })?;
        Ok(Self { raw })
    }

    /// `PaddingHadamard::try_from_parts(signs, padded_dim, subsample)` (padding_hadamard.rs:137-173).
    pub fn padding_hadamard(signs: &[bool], padded_dim: usize, subsample: Option<&[u32]>) -> Result<Self> {
        Self::create(sys::DAB_TRANSFORM_PADDING_HADAMARD, signs, padded_dim, None, subsample)
    }

    /// `DoubleHadamard::try_from_parts(signs0, signs1, subsample)` (double_hadamard.rs:146-206).
    pub fn double_hadamard(signs0: &[bool], signs1: &[bool], subsample: Option<&[u32]>) -> Result<Self> {
        Self::create(sys::DAB_TRANSFORM_DOUBLE_HADAMARD, signs0, signs1.len(), Some(signs1), subsample)
    }

    pub fn input_dim(&self) -> usize {
        unsafe { sys::dab_transform_input_dim(self.raw) as usize }
    }

    pub fn output_dim(&self) -> usize {
        unsafe { sys::dab_transform_output_dim(self.raw) as usize }
    }

    /// `transform_into` for `src.len() / input_dim` rows, on the device: `[n][output_dim]`.
    pub fn apply(&self, device: i32, src: &[f32]) -> Result<Vec<f32>> {
        let n = src.len() / self.input_dim().max(1);
        let mut out = vec![0f32; n * self.output_dim()];
        check(unsafe { sys::dab_transform_apply(self.raw, device, src.as_ptr(), n as u64, out.as_mut_ptr()) })?;
        Ok(out)
    }
}

impl Drop for Transform {
    fn drop(&mut self) {
        unsafe { sys::dab_transform_destroy(self.raw) }
    }
}

/// `MinMaxQuantizer::new(transform, grid_scale)` + `compress_into`: rows of `output_dim` codes, `Err` when a
/// transformed vector holds NaN (`InputContainsNaN`).
pub fn minmax_compress_transformed(transform: &Transform, device: i32, grid_scale: f32, nbits: i32, vectors: &[f32]) -> Result<(Vec<u8>, Vec<f32>)> {
    let n = vectors.len() / transform.input_dim().max(1);
    let row_bytes = unsafe { sys::dab_minmax_row_bytes(transform.output_dim() as u32, nbits) } as usize;
    let mut rows = vec![0u8; n * row_bytes];
    let mut loss = vec![0f32; n];
    check(unsafe {
        sys::dab_minmax_compress_transformed(transform.raw, device, grid_scale, nbits, vectors.as_ptr(), n as u64, rows.as_mut_ptr(), loss.as_mut_ptr())
    })?;
    Ok((rows, loss))
}

/// Full-precision queries behind `transform` against rows compressed behind it: `[nq][n]`.  `Err` when an
/// untransformed query holds NaN.
pub fn minmax_query_distances_transformed(transform: &Transform, device: i32, metric: Metric, nbits: i32, queries: &[f32], rows: &[u8]) -> Result<Vec<f32>> {
    let nq = queries.len() / transform.input_dim().max(1);
    let n = rows.len() / unsafe { sys::dab_minmax_row_bytes(transform.output_dim() as u32, nbits) } as usize;
    let mut out = vec![0f32; nq * n];
    check(unsafe {
        sys::dab_minmax_query_distances_transformed(transform.raw, device, metric as i32, nbits, queries.as_ptr(), nq as u32, rows.as_ptr(), n as u64, out.as_mut_ptr())
    })?;
    Ok(out)
}
