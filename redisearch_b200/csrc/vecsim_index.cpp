// Host logic of the device FLAT index.  See vecsim_index.h for the reference files mirrored.
#include "vecsim_index.h"
#include "batch_scratch.h"
#include "host_numeric.h"
#include "topk_common.cuh"
#include "coarse_tc.h"
#include "micro_batcher.h"

#include <algorithm>
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <chrono>
#include <limits>
#include <thread>

namespace rsb200 {

Globals &globals() {
    static Globals g;
    return g;
}

#define CU_OK(expr)                                                                                 \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            fprintf(stderr, "[vecsim_b200] CUDA error %s at %s:%d: %s\n", cudaGetErrorName(_e), __FILE__, __LINE__,  \
                    cudaGetErrorString(_e));                                                        \
            return false;                                                                           \
        }                                                                                           \
    } while (0)

// ------------------------------------------------------------------------------------------------
// QueryCtx
// ------------------------------------------------------------------------------------------------
QueryCtx::~QueryCtx() {
    if (stream) cudaStreamSynchronize(stream);
    cudaFree(d_query);
    cudaFreeHost(h_query);
    cudaFree(d_cand);
    cudaFree(d_out);
    cudaFreeHost(h_out);
    cudaFree(d_scores);
    cudaFree(d_count);
    cudaFreeHost(h_count);
    cudaFreeHost(h_abort);
    cudaFree(d_ids);
    cudaFreeHost(h_ids);
    cudaFree(d_dist);
    cudaFreeHost(h_dist);
    cudaFree(d_lab);
    if (ev_start) cudaEventDestroy(ev_start);
    if (ev_stop) cudaEventDestroy(ev_stop);
    if (stream) cudaStreamDestroy(stream);
}
bool QueryCtx::init() {
    CU_OK(cudaStreamCreateWithFlags(&stream, cudaStreamNonBlocking));
    CU_OK(cudaEventCreate(&ev_start));
    CU_OK(cudaEventCreate(&ev_stop));
    CU_OK(cudaMalloc(&d_count, 16));
    CU_OK(cudaMallocHost(&h_count, 16));
    CU_OK(cudaHostAlloc(&h_abort, 64, cudaHostAllocMapped));
    *h_abort = 0;
    void *dp = nullptr;
    CU_OK(cudaHostGetDevicePointer(&dp, h_abort, 0));
    d_abort = static_cast<const uint32_t *>(dp);
    return true;
}
template <class T> bool QueryCtx::grow(T *&d, size_t &cap, size_t new_cap, T **h) {
    cudaStreamSynchronize(stream);
    cudaFree(d);
    d = nullptr;
    if (h) {
        cudaFreeHost(*h);
        *h = nullptr;
    }
    cap = 0;
    CU_OK(cudaMalloc(&d, new_cap * sizeof(T)));
    if (h) CU_OK(cudaMallocHost(h, new_cap * sizeof(T)));
    cap = new_cap;
    return true;
}
bool QueryCtx::need_query(size_t bytes) {
    return bytes <= query_cap || grow(d_query, query_cap, std::max<size_t>(bytes, 64 * 1024), &h_query);
}
bool QueryCtx::need_cand(size_t elems) { return elems <= cand_cap || grow(d_cand, cand_cap, std::max<size_t>(elems, 64 * 1024)); }
bool QueryCtx::need_out(size_t elems) { return elems <= out_cap || grow(d_out, out_cap, std::max<size_t>(elems, 4096), &h_out); }
bool QueryCtx::need_scores(size_t n) { return n <= scores_cap || grow(d_scores, scores_cap, n + n / 8 + 1024); }
bool QueryCtx::need_ids(size_t n) { // ids and distances share one capacity
    const size_t cap = std::max<size_t>(n, 1024);
    return n <= ids_cap || (grow(d_ids, ids_cap, cap, &h_ids) && grow(d_dist, ids_cap, cap, &h_dist));
}
bool QueryCtx::need_lab(size_t elems) { return elems <= lab_cap || grow(d_lab, lab_cap, std::max<size_t>(elems, 64 * 1024)); }

// ------------------------------------------------------------------------------------------------
// construction
// ------------------------------------------------------------------------------------------------
static size_t elem_size(VecSimType t) {
    switch (t) {
    case VecSimType_FLOAT32: return 4;
    case VecSimType_FLOAT16:
    case VecSimType_BFLOAT16: return 2;
    case VecSimType_INT8:
    case VecSimType_UINT8: return 1;
    default: return 0;
    }
}

void FlatIndex::log(const char *level, const char *fmt, ...) const {
    logCallbackFunction cb = globals().log_cb.load();
    if (!cb) return;
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof(buf), fmt, ap);
    va_end(ap);
    cb(log_ctx_, level, buf);
}

FlatIndex *FlatIndex::create(const BFParams &p, void *log_ctx) {
    const size_t es = elem_size(p.type);
    if (es == 0 || p.dim == 0) return nullptr;
    int ndev = 0;
    if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= 0) {
        logCallbackFunction cb = globals().log_cb.load();
        const char *msg = "vecsim_b200: no CUDA device available; this library has no CPU fallback";
        if (cb)
            cb(log_ctx, "warning", msg);
        else
            fprintf(stderr, "%s\n", msg);
        cudaGetLastError();
        return nullptr;
    }
    std::unique_ptr<FlatIndex> ix(new FlatIndex());
    ix->type_ = p.type;
    ix->metric_ = p.metric;
    ix->dim_ = p.dim;
    ix->multi_ = p.multi;
    ix->block_size_ = p.blockSize ? p.blockSize : DEFAULT_BLOCK_SIZE;
    ix->log_ctx_ = log_ctx;
    ix->elem_bytes_ = es;
    switch (p.type) {
    case VecSimType_FLOAT32: ix->dtype_ = DT_F32; break;
    case VecSimType_FLOAT16: ix->dtype_ = DT_F16; break;
    case VecSimType_BFLOAT16: ix->dtype_ = DT_BF16; break;
    case VecSimType_INT8: ix->dtype_ = DT_I8; break;
    default: ix->dtype_ = DT_U8; break;
    }
    const bool is_int = (ix->dtype_ == DT_I8 || ix->dtype_ == DT_U8);
    ix->mkind_ = (p.metric == VecSimMetric_L2) ? MT_L2 : (p.metric == VecSimMetric_IP || !is_int) ? MT_IP : MT_COS;
    ix->stored_bytes_ = p.dim * es + ((is_int && p.metric == VecSimMetric_Cosine) ? sizeof(float) : 0);
    // fp32 rows are read with 4-byte lane loads (any dim); the narrower types with 16-byte vectors.
    ix->pitch_ = (ix->dtype_ == DT_F32) ? ix->stored_bytes_ : ((ix->stored_bytes_ + 15) & ~(size_t)15);
    if (cudaStreamCreateWithFlags(&ix->copy_stream_, cudaStreamNonBlocking) != cudaSuccess) return nullptr;
    // pinned staging: up to 32 MiB of appended rows between flushes
    ix->stage_cap_rows_ = std::max<size_t>(1, std::min<size_t>((32u << 20) / ix->pitch_, 1u << 20));
    if (cudaMallocHost(&ix->h_stage_, ix->stage_cap_rows_ * ix->pitch_) != cudaSuccess) return nullptr;
    memset(ix->h_stage_, 0, ix->stage_cap_rows_ * ix->pitch_);
    if (p.initialCapacity && !ix->reserve(p.initialCapacity)) return nullptr;
    return ix.release();
}

FlatIndex::~FlatIndex() {
    {
        std::lock_guard<std::mutex> g(pool_mu_);
        pool_.clear();
    }
    if (copy_stream_) {
        cudaStreamSynchronize(copy_stream_);
        cudaStreamDestroy(copy_stream_);
    }
    cudaFree(d_rows_);
    cudaFree(d_shadow_);
    cudaFree(d_shadow8_);
    cudaFree(d_tscale_);
    cudaFree(d_stats8_);
    cudaFree(d_norm2_);
    cudaFree(d_stats_);
    cudaFree(d_label_to_id_);
    cudaFree(d_label_rows_);
    cudaFree(d_id_to_label_);
    cudaFreeHost(h_stage_);
    for (TableSlot &t : table_ring_) {
        cudaEventSynchronize(t.ev);
        cudaEventDestroy(t.ev);
        cudaFreeHost(t.h);
    }
}

CorpusView FlatIndex::view() const {
    CorpusView v;
    v.rows = d_rows_;
    v.pitch = pitch_;
    v.n_rows = (uint32_t)count_;
    v.dim = (uint32_t)dim_;
    v.dtype = dtype_;
    v.metric = mkind_;
    return v;
}

std::unique_ptr<QueryCtx> FlatIndex::checkout() {
    {
        std::unique_lock<std::mutex> g(pool_mu_);
        if (!pool_.empty()) {
            auto c = std::move(pool_.back());
            pool_.pop_back();
            g.unlock();
            if (c->abandoned) { // its last user timed out and left: let that work drain before the buffers are reused
                cudaStreamSynchronize(c->stream);
                c->abandoned = false;
                *c->h_abort = 0;
            }
            return c;
        }
    }
    std::unique_ptr<QueryCtx> c(new QueryCtx());
    if (!c->init()) return nullptr;
    return c;
}
void FlatIndex::checkin(std::unique_ptr<QueryCtx> c) {
    if (!c) return;
    std::lock_guard<std::mutex> g(pool_mu_);
    if (pool_.size() < 64) pool_.push_back(std::move(c));
}

bool FlatIndex::timed_out(void *ctx) const {
    timeoutCallbackFunction cb = globals().timeout_cb.load();
    return cb && cb(ctx) != 0;
}

int FlatIndex::wait_polling(cudaStream_t s, void *timeout_ctx) const {
    timeoutCallbackFunction cb = globals().timeout_cb.load();
    if (!cb) return cudaStreamSynchronize(s) == cudaSuccess ? 0 : -1;
    for (;;) {
        const cudaError_t e = cudaStreamQuery(s);
        if (e == cudaSuccess) return 0;
        if (e != cudaErrorNotReady) return -1;
        if (cb(timeout_ctx) != 0) return 1;
        std::this_thread::sleep_for(std::chrono::microseconds(50));
    }
}

int FlatIndex::wait_or_abandon(QueryCtx &c, void *timeout_ctx) const {
    const int w = wait_polling(c.stream, timeout_ctx);
    if (w == 1) { // the next checkout synchronises before the buffers are reused
        c.abandoned = true;
        *c.h_abort = 1;
    }
    return w;
}

void FlatIndex::record_scan(const QueryCtx *c, uint64_t bytes) {
    float ms = 0;
    if (c && cudaEventElapsedTime(&ms, c->ev_start, c->ev_stop) != cudaSuccess) return;
    std::lock_guard<std::mutex> g(stats_mu_);
    scan_us_ += ms * 1000.0;
    scan_launches_++;
    scan_bytes_ += bytes;
}

// ------------------------------------------------------------------------------------------------
// preprocessing (VS/spaces/computer/preprocessors.h:49-146)
// ------------------------------------------------------------------------------------------------
void FlatIndex::preprocess_storage(const void *blob, uint8_t *dst) const {
    memcpy(dst, blob, dim_ * elem_bytes_);
    if (metric_ != VecSimMetric_Cosine) return;
    switch (dtype_) {
    case DT_F32: normalize_f32(reinterpret_cast<float *>(dst), dim_); break;
    case DT_F16: normalize_f16(reinterpret_cast<uint16_t *>(dst), dim_); break;
    case DT_BF16: normalize_bf16(reinterpret_cast<uint16_t *>(dst), dim_); break;
    case DT_I8: append_int_norm(reinterpret_cast<int8_t *>(dst), dim_); break;
    case DT_U8: append_int_norm(reinterpret_cast<uint8_t *>(dst), dim_); break;
    }
}
void FlatIndex::preprocess_query(const void *blob, uint8_t *dst) const { preprocess_storage(blob, dst); }

// ------------------------------------------------------------------------------------------------
// storage
// ------------------------------------------------------------------------------------------------
bool FlatIndex::grow_to(size_t rows) {
    if (rows <= capacity_) return true;
    size_t cap = std::max(rows, capacity_ + capacity_ / 2);
    cap = ((cap + block_size_ - 1) / block_size_) * block_size_;
    uint8_t *nu = nullptr;
    cudaError_t e = cudaMalloc(&nu, cap * pitch_);
    if (e != cudaSuccess && cap > rows) { // retry with the exact size
        cudaGetLastError();
        cap = ((rows + block_size_ - 1) / block_size_) * block_size_;
        e = cudaMalloc(&nu, cap * pitch_);
    }
    if (e != cudaSuccess) {
        cudaGetLastError();
        log("warning", "vecsim_b200: cannot allocate %zu bytes of HBM", cap * pitch_);
        return false;
    }
    if (resident_) {
        CU_OK(cudaMemcpyAsync(nu, d_rows_, resident_ * pitch_, cudaMemcpyDeviceToDevice, copy_stream_));
        CU_OK(cudaStreamSynchronize(copy_stream_));
    }
    cudaFree(d_rows_);
    d_rows_ = nu;
    capacity_ = cap;
    return true;
}

bool FlatIndex::reserve(size_t rows) {
    std::lock_guard<std::mutex> g(mu_);
    if (id_to_label_.capacity() < rows) id_to_label_.reserve(rows);
    return grow_to(rows);
}

// caller holds mu_
static bool flush_locked(uint8_t *d_rows, size_t pitch, uint8_t *h_stage, size_t &resident, size_t count,
                         cudaStream_t s) {
    if (resident == count) return true;
    const size_t n = count - resident;
    CU_OK(cudaMemcpyAsync(d_rows + resident * pitch, h_stage, n * pitch, cudaMemcpyHostToDevice, s));
    CU_OK(cudaStreamSynchronize(s));
    resident = count;
    return true;
}

bool FlatIndex::flush() {
    std::lock_guard<std::mutex> g(mu_);
    return flush_locked(d_rows_, pitch_, h_stage_, resident_, count_, copy_stream_);
}

int FlatIndex::add(const void *blob, size_t label) {
    std::lock_guard<std::mutex> g(mu_);
    if (!multi_) {
        auto it = label_to_id_.find(label);
        if (it != label_to_id_.end()) {
            // brute_force_single.h:139-144: overwrite in place with the RAW blob (the reference does
            // not re-run the storage preprocessor here).  For int8/uint8 cosine the reference reads
            // 4 bytes past the caller's blob; we recompute the norm instead of reading out of bounds.
            const idType id = it->second;
            std::vector<uint8_t> tmp(pitch_, 0);
            memcpy(tmp.data(), blob, dim_ * elem_bytes_);
            if (mkind_ == MT_COS) {
                if (dtype_ == DT_I8)
                    append_int_norm(reinterpret_cast<int8_t *>(tmp.data()), dim_);
                else
                    append_int_norm(tmp.data(), dim_);
            }
            if (id >= resident_) {
                memcpy(h_stage_ + (id - resident_) * pitch_, tmp.data(), pitch_);
            } else {
                if (cudaMemcpy(d_rows_ + (size_t)id * pitch_, tmp.data(), pitch_, cudaMemcpyHostToDevice) != cudaSuccess)
                    return 0;
                if (keeps_row_copies()) shadow_dirty_.push_back(id);
            }
            // the overwritten row is the caller's RAW blob: a cosine index may now hold a non-unit row, so the coarse
            // proof must stop assuming unit vectors (it switches to the norm-scaled bound of the inner-product route)
            if (metric_ == VecSimMetric_Cosine && dtype_ == DT_F32 && !raw_rows_) {
                raw_rows_ = true;
                shadow_rows_ = 0; // |row|^2 and the running maxima have to be built for every row
                shadow_dirty_.clear();
            }
            return 0;
        }
    }
    if (count_ >= (size_t)std::numeric_limits<uint32_t>::max() - 1) return 0;
    if (count_ - resident_ >= stage_cap_rows_) {
        if (!grow_to(count_ + 1)) return 0;
        if (!flush_locked(d_rows_, pitch_, h_stage_, resident_, count_, copy_stream_)) return 0;
    }
    if (!grow_to(count_ + 1)) return 0;
    uint8_t *slot = h_stage_ + (count_ - resident_) * pitch_;
    preprocess_storage(blob, slot);
    const idType id = (idType)count_++;
    id_to_label_.push_back(label);
    if (multi_) {
        auto &ids = label_to_ids_[label];
        label_rows_changed(ids.size(), ids.size() + 1);
        ids.push_back(id);
    } else {
        label_to_id_[label] = id;
    }
    labels_dirty_ = true;
    l2i_dirty_ = true;
    return 1;
}

int FlatIndex::add_bulk(const void *blobs, size_t stride, size_t n, const size_t *labels, size_t label0) {
    int added = 0;
    for (size_t i = 0; i < n; i++)
        added += add(static_cast<const uint8_t *>(blobs) + i * stride, labels ? labels[i] : label0 + i);
    return added;
}

int FlatIndex::add_bulk_device(const void *d_src, size_t n, size_t label0) {
    std::lock_guard<std::mutex> g(mu_);
    if (n == 0) return 0;
    if (!flush_locked(d_rows_, pitch_, h_stage_, resident_, count_, copy_stream_)) return -1;
    if (!grow_to(count_ + n)) return -1;
    if (cudaMemcpyAsync(d_rows_ + count_ * pitch_, d_src, n * pitch_, cudaMemcpyDeviceToDevice, copy_stream_) !=
            cudaSuccess ||
        cudaStreamSynchronize(copy_stream_) != cudaSuccess)
        return -1;
    id_to_label_.reserve(count_ + n);
    for (size_t i = 0; i < n; i++) {
        const idType id = (idType)(count_ + i);
        id_to_label_.push_back(label0 + i);
        if (multi_) {
            auto &ids = label_to_ids_[label0 + i];
            label_rows_changed(ids.size(), ids.size() + 1);
            ids.push_back(id);
        } else {
            label_to_id_[label0 + i] = id;
        }
    }
    count_ += n;
    resident_ = count_;
    labels_dirty_ = true;
    l2i_dirty_ = true;
    return (int)n;
}

int FlatIndex::remove(size_t label) {
    std::lock_guard<std::mutex> g(mu_);
    std::vector<idType> victims;
    if (multi_) {
        auto it = label_to_ids_.find(label);
        if (it == label_to_ids_.end()) return 0;
        victims = it->second;
        label_to_ids_.erase(it);
        label_rows_changed(victims.size(), 0);
    } else {
        auto it = label_to_id_.find(label);
        if (it == label_to_id_.end()) return 0;
        victims.push_back(it->second);
        label_to_id_.erase(it);
    }
    if (!flush_locked(d_rows_, pitch_, h_stage_, resident_, count_, copy_stream_)) return 0;
    // brute_force.h:196-224 — move the last row into the hole; with several victims process them
    // one by one (brute_force_multi.h:143-165), re-reading ids that a previous swap relocated.
    int removed = 0;
    std::sort(victims.begin(), victims.end(), std::greater<idType>());
    for (idType id : victims) {
        const idType last = (idType)(count_ - 1);
        if (id != last) {
            const size_t last_label = id_to_label_[last];
            cudaMemcpyAsync(d_rows_ + (size_t)id * pitch_, d_rows_ + (size_t)last * pitch_, pitch_,
                            cudaMemcpyDeviceToDevice, copy_stream_);
            if (keeps_row_copies()) shadow_dirty_.push_back(id);
            id_to_label_[id] = last_label;
            if (multi_) {
                auto &v = label_to_ids_[last_label];
                for (auto &x : v)
                    if (x == last) x = id;
            } else {
                label_to_id_[last_label] = id;
            }
        }
        id_to_label_.pop_back();
        count_--;
        removed++;
    }
    // row ids >= count_ will be re-used by later appends: the shadow copy (and |row|^2) of those ids is stale
    shadow_rows_ = std::min(shadow_rows_, count_);
    cudaStreamSynchronize(copy_stream_);
    resident_ = count_;
    labels_dirty_ = true;
    l2i_dirty_ = true;
    return removed;
}

void FlatIndex::label_rows_changed(size_t from, size_t to) {
    if (from) {
        auto it = rows_per_label_.find(from);
        if (it != rows_per_label_.end() && --it->second == 0) rows_per_label_.erase(it);
    }
    if (to) rows_per_label_[to]++;
}

size_t FlatIndex::max_rows_per_label() const {
    std::lock_guard<std::mutex> g(mu_);
    return rows_per_label_.empty() ? 0 : rows_per_label_.rbegin()->first;
}

bool FlatIndex::read_rows(size_t first, size_t n, void *host_dst) {
    if (!flush()) return false;
    if (first + n > count_ || !host_dst) return false;
    if (n == 0) return true;
    return cudaMemcpy2D(host_dst, stored_bytes_, d_rows_ + first * pitch_, pitch_, stored_bytes_, n, cudaMemcpyDeviceToHost) == cudaSuccess;
}

bool FlatIndex::sync_labels_to_device() {
    std::lock_guard<std::mutex> g(mu_);
    if (!labels_dirty_ && d_id_to_label_) return true;
    if (count_ > d_labels_cap_) {
        cudaFree(d_id_to_label_);
        d_id_to_label_ = nullptr;
        const size_t cap = std::max(capacity_, count_);
        CU_OK(cudaMalloc(&d_id_to_label_, cap * sizeof(uint64_t)));
        d_labels_cap_ = cap;
    }
    static_assert(sizeof(size_t) == sizeof(uint64_t), "labels are 64-bit");
    if (count_)
        CU_OK(cudaMemcpy(d_id_to_label_, id_to_label_.data(), count_ * sizeof(uint64_t), cudaMemcpyHostToDevice));
    labels_dirty_ = false;
    return true;
}

// ------------------------------------------------------------------------------------------------
// queries
// ------------------------------------------------------------------------------------------------
bool FlatIndex::stage_queries(QueryCtx &c, const void *blobs, size_t stride, size_t nq, bool raw, const void *tail, size_t tail_bytes) {
    const size_t qp = query_pitch(), bytes = qp * nq + tail_bytes;
    if (!c.need_query(bytes)) return false;
    memset(c.h_query, 0, qp * nq);
    for (size_t i = 0; i < nq; i++) {
        const uint8_t *blob = static_cast<const uint8_t *>(blobs) + i * stride;
        if (raw)
            preprocess_query(blob, c.h_query + i * qp);
        else
            memcpy(c.h_query + i * qp, blob, stored_bytes_);
    }
    if (tail_bytes) memcpy(c.h_query + qp * nq, tail, tail_bytes);
    CU_OK(cudaMemcpyAsync(c.d_query, c.h_query, bytes, cudaMemcpyHostToDevice, c.stream));
    return true;
}

// composite (score key << 32 | row) -> the row's label (from `id_to_label`) and its score
static VecSimQueryResult decode(uint64_t comp, const std::vector<size_t> &id_to_label) {
    return {id_to_label[(uint32_t)comp], (double)key_to_float((uint32_t)(comp >> 32))};
}

// reply ordering: (score asc, label asc) — the order the reference's heap drains in
// (vecsim_stl.h:64-84) — or by label (vec_utils.cpp:100-103).
void FlatIndex::finish_reply(VecSimQueryReply *rep, VecSimQueryReply_Order order) const {
    auto &r = rep->results;
    if (order == BY_ID) {
        std::sort(r.begin(), r.end(), [](const VecSimQueryResult &a, const VecSimQueryResult &b) { return a.id < b.id; });
    } else {
        std::sort(r.begin(), r.end(), [](const VecSimQueryResult &a, const VecSimQueryResult &b) {
            const bool an = std::isnan(a.score), bn = std::isnan(b.score);
            if (an != bn) return bn; // NaN last
            if (!an && a.score != b.score) return a.score < b.score;
            return a.id < b.id;
        });
    }
}

long FlatIndex::select_from_scores(QueryCtx &c, uint32_t n, bool has_cursor, uint64_t cursor, size_t want) {
    if (want == 0 || n == 0) return 0;
    if (!c.need_out(want + 1)) return -1;
    LaunchCounters lc;
    const uint64_t *cur_ptr = nullptr;
    if (has_cursor) {
        *reinterpret_cast<uint64_t *>(c.h_count) = cursor;
        if (cudaMemcpyAsync(c.d_out + want, c.h_count, 8, cudaMemcpyHostToDevice, c.stream) != cudaSuccess) return -1;
        cur_ptr = c.d_out + want;
    }
    const uint32_t lists = plan_select_scores_lists(n);
    size_t found = 0;
    while (found < want) {
        const uint32_t chunk = (uint32_t)std::min<size_t>(kMaxFusedK, want - found);
        if (!c.need_cand((size_t)lists * chunk)) return -1;
        if (launch_select_scores(c.d_scores, n, cur_ptr, chunk, c.d_cand, c.stream, &lc) != cudaSuccess) return -1;
        if (launch_final_select(c.d_cand, 1, lists * chunk, chunk, c.d_out + found, c.stream, &lc) != cudaSuccess)
            return -1;
        found += chunk;
        cur_ptr = c.d_out + found - 1;
    }
    if (cudaMemcpyAsync(c.h_out, c.d_out, want * 8, cudaMemcpyDeviceToHost, c.stream) != cudaSuccess) return -1;
    if (cudaStreamSynchronize(c.stream) != cudaSuccess) return -1;
    launches_total_ += lc.launches;
    size_t real = 0;
    while (real < want && c.h_out[real] != kEmptySlot) real++;
    return (long)real;
}

VecSimQueryReply *FlatIndex::topk(const void *q, size_t k, VecSimQueryParams *qp, VecSimQueryReply_Order order) {
    auto *rep = new VecSimQueryReply();
    last_mode_ = STANDARD_KNN;
    void *tctx = qp ? qp->timeoutCtx : nullptr;
    if (k == 0) return rep; // brute_force.h:251-253
    if (!flush()) return rep;
    const size_t n = count_;
    if (n == 0) return rep;
    if (timed_out(tctx)) {
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    auto c = checkout();
    if (!c) return rep;
    const size_t qpitch = query_pitch();
    bool ok = stage_queries(*c, q, 0, 1, true);
    const CorpusView v = view();
    LaunchCounters lc;
    if (ok && !multi_ && std::min(k, n) <= (size_t)kMaxFusedK) {
        const uint32_t ke = (uint32_t)std::min(k, n);
        const uint64_t *d_res = nullptr;
        if (single_query_takes_coarse(ke, reinterpret_cast<const float *>(c->h_query), q8_route(1, ke))) {
            // an up-to-date fp16 shadow exists (a batch built it): one pass over 15 GB of it + exact rescoring + proof
            // beats the 31 GB exact scan; same answer (DESIGN.md §4)
            uint64_t *r = nullptr;
            ok = batch_scan(*c, c->d_query, qpitch, 1, ke, c->stream, lc, &r);
            d_res = r;
        } else {
            last_batch_path_ = 0;
            const ScanPlan plan = plan_scan_topk(v, 1, ke);
            ok = c->need_cand(plan.cand_elems) && c->need_out(ke);
            if (ok) {
                cudaEventRecord(c->ev_start, c->stream);
                ok = launch_scan_topk(v, c->d_query, qpitch, 1, ke, plan, c->d_cand, c->stream, &lc, nullptr, c->d_abort) == cudaSuccess;
                cudaEventRecord(c->ev_stop, c->stream);
            }
            ok = ok && launch_final_select(c->d_cand, 1, plan.lists_per_query * ke, ke, c->d_out, c->stream, &lc) == cudaSuccess;
            d_res = c->d_out;
        }
        ok = ok && cudaMemcpyAsync(c->h_out, d_res, ke * 8, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess;
        if (ok) {
            const int w = wait_or_abandon(*c, tctx);
            if (w == 1) { // deadline passed while the scan was running
                launches_total_ += lc.launches;
                checkin(std::move(c));
                rep->code = VecSim_QueryReply_TimedOut;
                return rep;
            }
            ok = w == 0;
        }
        if (ok) {
            record_scan(c.get(), (uint64_t)n * stored_bytes_);
            for (uint32_t i = 0; i < ke && c->h_out[i] != kEmptySlot; i++)
                rep->results.push_back(decode(c->h_out[i], id_to_label_));
        }
    } else if (ok) {
        // k > kMaxFusedK or multi-value: materialise all scores, then cursor-select in chunks.
        ok = c->need_scores(n);
        if (ok) {
            cudaEventRecord(c->ev_start, c->stream);
            ok = launch_scan_scores(v, c->d_query, c->d_scores, c->stream, &lc) == cudaSuccess;
            cudaEventRecord(c->ev_stop, c->stream);
        }
        if (ok) {
            const size_t want_labels = std::min(k, label_count());
            bool has_cursor = false;
            uint64_t cursor = 0;
            std::unordered_set<size_t> seen;
            size_t scanned = 0;
            while (ok && rep->results.size() < want_labels && scanned < n) {
                const size_t want = multi_ ? std::min<size_t>(std::max<size_t>(2 * (want_labels - rep->results.size()), 64), n - scanned)
                                           : std::min(want_labels - rep->results.size(), n - scanned);
                const long got = select_from_scores(*c, (uint32_t)n, has_cursor, cursor, want);
                if (got < 0) {
                    ok = false;
                    break;
                }
                for (long i = 0; i < got && rep->results.size() < want_labels; i++) {
                    const VecSimQueryResult r = decode(c->h_out[i], id_to_label_);
                    if (multi_ && !seen.insert(r.id).second) continue; // best score per label comes first
                    rep->results.push_back(r);
                }
                scanned += (size_t)got;
                if ((size_t)got < want) break;
                has_cursor = true;
                cursor = c->h_out[got - 1];
            }
            if (ok) record_scan(c.get(), (uint64_t)n * stored_bytes_);
        }
    }
    launches_total_ += lc.launches;
    if (!ok) {
        log("warning", "vecsim_b200: top-k query failed on device");
        rep->results.clear();
    }
    checkin(std::move(c));
    if (timed_out(tctx)) {
        rep->results.clear();
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    finish_reply(rep, order);
    return rep;
}

// -1 = from env VECSIM_B200_COARSE (default 1), 0 = exact scans only, 1 = fp16 shadow rows, 2 = TF32 on the fp32 rows
std::atomic<int> g_coarse_mode{-1};

// second tier of the coarse route (lists of 128 for the queries the first proof left open); VECSIM_B200_TIER2=0 turns it off
static bool coarse_tier2_enabled() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("VECSIM_B200_TIER2");
        v = (e && atoi(e) == 0) ? 0 : 1;
    }
    return v != 0;
}

// two-pass first tier of the fp16 route (sample pass -> fixed admission bound -> main pass); VECSIM_B200_FIXED=0 falls back
// to the single pass with adaptive lists
static bool coarse_fixed_enabled() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("VECSIM_B200_FIXED");
        v = (e && atoi(e) == 0) ? 0 : 1;
    }
    return v != 0;
}

static int coarse_mode() {
    int m = g_coarse_mode.load();
    if (m < 0) {
        const char *e = getenv("VECSIM_B200_COARSE");
        m = e ? atoi(e) : 1;
        if (m < 0 || m > 2) m = 1;
        g_coarse_mode.store(m);
    }
    return m;
}

// Single queries (and batches below 16) take the tensor-core route only if that costs nothing extra: mode 1, the copy the route
// reads already complete, fp32 cosine, k within the coarse lists.  host_query (nullable): the stored-form query; a raw
// inner-product / L2 query whose fp16 form is not finite (|x| >= 65520 or NaN) cannot be proven and takes the exact scan.  q8:
// the route reads the int8 copy (KNN batches where q8_route holds), else the fp16 shadow (every other KNN batch, and the range
// and hybrid routes).
bool FlatIndex::single_query_takes_coarse(uint32_t ke, const float *host_query, bool q8) {
    if (coarse_mode() != 1 || multi_ || coarse_disabled_ || dtype_ != DT_F32) return false;
    if (!unit_rows() && !(shadow_max_abs_ <= 60000.0f)) return false; // fp16 range (also false before the first build)
    if (!unit_rows() && host_query)
        for (size_t i = 0; i < dim_; i++)
            if (!(std::fabs(host_query[i]) < 65520.0f)) return false;
    {
        std::lock_guard<std::mutex> g(mu_);
        if (!(q8 ? d_shadow8_ && std::isfinite(shadow8_delta_) && std::isfinite(shadow8_xmax_) : d_shadow_ != nullptr) ||
            shadow_rows_ != count_ || !shadow_dirty_.empty() || shadow_cap_ < count_)
            return false;
    }
    return q8 || coarse_supported(view(), 1, ke, CoarseF16);
}

bool FlatIndex::q8_route(uint32_t nq, uint32_t ke) const {
    return coarse_mode() == 1 && !multi_ && unit_rows() && coarse_fixed_enabled() && coarse_supported(view(), nq, ke, CoarseQ8);
}

// Bring the fp16 shadow copy of the rows up to date on `st` (rows appended, overwritten or moved by a
// swap-delete since the last coarse batch).  Returns false if HBM for the shadow cannot be had; the
// caller then runs the TF32 variant on the fp32 rows.
// int8 / uint8 L2 indexes keep no shadow, only the exact int32 |row|^2 of every row, under the same bookkeeping.  fp16 / bf16
// indexes keep no shadow either, only |row|^2 of the stored rows and its running maximum (the direct range route's X).
bool FlatIndex::ensure_shadow(cudaStream_t st, bool q8) {
    std::lock_guard<std::mutex> g(mu_);
    const bool inorm = int_l2(), rows16 = dtype_ == DT_F16 || dtype_ == DT_BF16;
    const bool norms_only = inorm || rows16;
    if (norms_only && (shadow_cap_ < count_ || !d_norm2_)) {
        const size_t cap = std::max(capacity_, count_);
        cudaFree(d_norm2_);
        d_norm2_ = nullptr;
        shadow_cap_ = shadow_rows_ = 0;
        shadow_dirty_.clear();
        if (cudaMalloc(&d_norm2_, cap * sizeof(int32_t)) != cudaSuccess) {
            cudaGetLastError();
            d_norm2_ = nullptr;
            return false;
        }
        shadow_cap_ = cap;
    }
    if (rows16 && !d_stats_ && (cudaMalloc(&d_stats_, 8) != cudaSuccess || cudaMemset(d_stats_, 0, 8) != cudaSuccess)) {
        cudaGetLastError();
        return false;
    }
    bool launched = false;
    if (!norms_only && shadow_cap_ >= count_ && (q8 ? !d_shadow8_ : !d_shadow_) && (d_shadow_ || d_shadow8_)) {
        // the other copy is kept: allocate only the missing one and build it over the rows the other covers; the refresh below
        // brings both over dirty and appended rows
        const size_t cap = shadow_cap_;
        uint8_t *nu = nullptr;
        float *nsc = nullptr;
        if (cudaMalloc(&nu, q8 ? coarse_shadow8_bytes((uint32_t)cap, (uint32_t)dim_) : coarse_shadow_bytes((uint32_t)cap, (uint32_t)dim_)) !=
                cudaSuccess ||
            (q8 && (cudaMalloc(&nsc, (cap + 127) / 128 * sizeof(float)) != cudaSuccess ||
                    (!d_stats8_ && cudaMalloc(&d_stats8_, 8) != cudaSuccess)))) {
            cudaGetLastError();
            cudaFree(nu);
            cudaFree(nsc);
            return false;
        }
        const uint32_t n = (uint32_t)std::min(shadow_rows_, count_);
        cudaError_t e;
        if (q8) {
            d_shadow8_ = nu;
            d_tscale_ = nsc;
            e = cudaMemsetAsync(d_stats8_, 0, 8, st);
            if (e == cudaSuccess) e = launch_to_i8_tiled(d_rows_, pitch_, (uint32_t)dim_, (uint32_t)count_, 0, n, d_shadow8_, d_tscale_, d_stats8_, st);
        } else {
            d_shadow_ = nu;
            e = launch_to_f16_tiled(d_rows_, pitch_, (uint32_t)dim_, 0, n, d_shadow_, st);
        }
        if (e != cudaSuccess) { // the new copy does not cover the rows: every copy is rebuilt next time
            shadow_rows_ = 0;
            shadow_dirty_.clear();
            return false;
        }
        launched = true;
    }
    if (!norms_only && (shadow_cap_ < count_ || (q8 ? !d_shadow8_ : !d_shadow_))) {
        // the requested copy and every copy already kept, at the capacity; rows are re-converted below
        const size_t cap = std::max(capacity_, count_);
        const bool k16 = !q8 || d_shadow_, k8 = q8 || d_shadow8_;
        uint8_t *nu = nullptr, *nu8 = nullptr;
        float *nsc = nullptr;
        if ((k16 && cudaMalloc(&nu, coarse_shadow_bytes((uint32_t)cap, (uint32_t)dim_)) != cudaSuccess) ||
            (k8 && (cudaMalloc(&nu8, coarse_shadow8_bytes((uint32_t)cap, (uint32_t)dim_)) != cudaSuccess ||
                    cudaMalloc(&nsc, (cap + 127) / 128 * sizeof(float)) != cudaSuccess)) ||
            (k8 && !d_stats8_ && cudaMalloc(&d_stats8_, 8) != cudaSuccess)) {
            cudaGetLastError();
            cudaFree(nu);
            cudaFree(nu8);
            cudaFree(nsc);
            return false;
        }
        cudaFree(d_shadow_);
        cudaFree(d_shadow8_);
        cudaFree(d_tscale_);
        d_shadow_ = nu;
        d_shadow8_ = nu8;
        d_tscale_ = nsc;
        cudaFree(d_norm2_);
        d_norm2_ = nullptr;
        shadow_cap_ = cap;
        shadow_rows_ = 0;
        shadow_dirty_.clear();
    }
    if (!norms_only && !unit_rows() && !d_norm2_) { // L2 / raw inner product / cosine after a raw overwrite: the error bound (and
                                                    // the L2 epilogue) need |row|^2 of every row
        if (!d_stats_ && (cudaMalloc(&d_stats_, 8) != cudaSuccess || cudaMemset(d_stats_, 0, 8) != cudaSuccess)) {
            cudaGetLastError();
            return false;
        }
        if (cudaMalloc(&d_norm2_, shadow_cap_ * sizeof(float)) != cudaSuccess) {
            cudaGetLastError();
            return false;
        }
        shadow_rows_ = 0;
        shadow_dirty_.clear();
    }
    if (shadow_rows_ > count_) shadow_rows_ = count_;
    // rows [first, first + n) into every copy this index keeps (the int8 copy re-quantizes the whole tiles that hold them: a
    // changed row may change its tile's scale)
    const auto refresh = [&](uint32_t first, uint32_t n) {
        if (inorm) return launch_int_norm2(d_rows_, pitch_, (uint32_t)dim_, first, n, dtype_ == DT_I8, reinterpret_cast<int32_t *>(d_norm2_), st) ==
                          cudaSuccess;
        if (d_shadow_ && launch_to_f16_tiled(d_rows_, pitch_, (uint32_t)dim_, first, n, d_shadow_, st) != cudaSuccess) return false;
        if (d_shadow8_ && launch_to_i8_tiled(d_rows_, pitch_, (uint32_t)dim_, (uint32_t)count_, first, n, d_shadow8_, d_tscale_, d_stats8_, st) !=
                              cudaSuccess)
            return false;
        return !d_norm2_ || launch_row_stats(d_rows_, pitch_, (uint32_t)dim_, first, n, d_norm2_, d_stats_, st, dtype_) == cudaSuccess;
    };
    if (shadow_dirty_.size() > 256) {
        shadow_rows_ = 0;
        shadow_dirty_.clear();
    }
    // a full rebuild recomputes the int8 copy's residual and norm maxima
    if (d_shadow8_ && shadow_rows_ == 0 && count_ > 0 && cudaMemsetAsync(d_stats8_, 0, 8, st) != cudaSuccess) return false;
    for (idType id : shadow_dirty_)
        if (id < shadow_rows_) {
            if (!refresh(id, 1)) return false;
            launched = true;
        }
    shadow_dirty_.clear();
    if (shadow_rows_ < count_) {
        if (!refresh((uint32_t)shadow_rows_, (uint32_t)(count_ - shadow_rows_))) return false;
        shadow_rows_ = count_;
        launched = true;
    }
    // other query streams may read the shadow as soon as the lock is released
    if (launched) {
        const bool stats = d_norm2_ && !inorm;
        uint32_t h[2] = {0, 0}, h8[2] = {0, 0};
        if (stats && cudaMemcpyAsync(h, d_stats_, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return false;
        if (d_shadow8_ && cudaMemcpyAsync(h8, d_stats8_, 8, cudaMemcpyDeviceToHost, st) != cudaSuccess) return false;
        if (cudaStreamSynchronize(st) != cudaSuccess) return false;
        if (d_shadow8_) {
            memcpy(&shadow8_delta_, &h8[0], 4);
            memcpy(&shadow8_xmax_, &h8[1], 4);
        }
        if (stats) { // running maxima over every row ever converted (deletes do not lower them: conservative)
            float n2, ma;
            memcpy(&n2, &h[0], 4);
            memcpy(&ma, &h[1], 4);
            shadow_max_norm_ = std::sqrt(n2);
            shadow_max_abs_ = ma;
        }
    }
    return true;
}

void FlatIndex::disable_coarse() {
    std::lock_guard<std::mutex> g(mu_);
    coarse_disabled_ = true;
    cudaFree(d_shadow_);
    cudaFree(d_shadow8_);
    cudaFree(d_tscale_);
    cudaFree(d_norm2_);
    d_shadow_ = nullptr;
    d_shadow8_ = nullptr;
    d_tscale_ = nullptr;
    d_norm2_ = nullptr;
    shadow_cap_ = shadow_rows_ = 0;
    shadow_dirty_.clear();
}

bool FlatIndex::shadow_values_in_range() {
    if (unit_rows() || shadow_max_abs_ <= 60000.0f) return true;
    disable_coarse(); // the shadow's HBM is given back
    return false;
}

bool FlatIndex::shadow_operands(const void *d_q, size_t qpitch, uint32_t nq, uint8_t *q16, float *d_qn2, cudaStream_t st, LaunchCounters &lc,
                                CoarseOperands &ops) {
    const size_t q16_pitch = f16_query_pitch();
    ops = CoarseOperands{d_shadow_, 0, q16, q16_pitch, 0, mkind_ == MT_L2 ? 1 : 0, d_norm2_, d_qn2};
    bool ok = launch_to_f16(d_q, qpitch, (uint32_t)dim_, 0, nq, q16, q16_pitch, st) == cudaSuccess;
    if (d_qn2) ok = ok && launch_row_stats(d_q, qpitch, (uint32_t)dim_, 0, nq, d_qn2, nullptr, st) == cudaSuccess;
    lc.launches += d_qn2 ? 2 : 1;
    return ok;
}

// int8 / uint8: s8 / u8 wgmma dot products are exact integers and the epilogue applies the reference's own float expression, so
// the 8-bit routes are bit-exact.  L2: |row|^2 + |q|^2 - 2 dot in int32, rounded once to float, is the reference's float(sum of
// squared differences) bit for bit
bool FlatIndex::direct8_operands(const void *d_q, size_t qpitch, uint32_t nq, int32_t *d_qn, cudaStream_t st, LaunchCounters &lc,
                                 CoarseOperands &ops) {
    ops = CoarseOperands{d_rows_, pitch_, d_q, qpitch, dtype_ == DT_I8 ? 1 : 0, mkind_ == MT_COS ? 1 : int_l2() ? 2 : 0, nullptr, nullptr};
    if (!int_l2()) return true;
    ops.row_norm2 = reinterpret_cast<const float *>(d_norm2_); // int32 values (CoarseOperands)
    ops.q_norm2 = reinterpret_cast<const float *>(d_qn);
    lc.launches++;
    return launch_int_norm2(d_q, qpitch, (uint32_t)dim_, 0, nq, dtype_ == DT_I8, d_qn, st) == cudaSuccess;
}

void FlatIndex::RangeScratch::take(BatchScratch &s, const FlatIndex &ix, CoarseKind kind, const CoarsePlan &cp, uint32_t nq, bool fold) {
    const bool shadow = kind == CoarseF16, refine = kind != CoarseDirect8; // refine: rescored by range_refine_kernel
    cand = s.take<uint64_t>((size_t)nq * cp.grid_x * cp.keep);
    list_scratch = s.take<uint64_t>(cp.scratch_elems);
    q16 = s.take<uint8_t>(shadow ? nq * ix.f16_query_pitch() : 0);
    qn2 = s.take<float>((shadow && !ix.unit_rows()) || (kind == CoarseDirect8 && ix.int_l2()) ? nq : 0); // |q|^2 (fp32), or int32 for 8-bit L2
    thr = s.take<float>(refine ? nq : 0);                 // bound of the main pass per query
    ovf = s.take<uint32_t>(nq);                           // a list of the main pass ran full
    front = s.take<uint32_t>(fold && refine ? nq : 0);    // multi-value: the hit rows at the front of each list segment
}

// CoarseF16: T_q = radius_q + eps_q over the fp16 shadow, then exact rescoring (DESIGN.md §4).  CoarseDirect16: the margin eps16_q
// over the stored rows and CUDA-core rescoring (§4.11).  CoarseDirect8: the radii themselves over exact integer distances, packed.
// Launches: 4 (+1 for |q|^2 of rows not all unit), 3, 2 (+1 for L2); one more for a fold after rescoring
bool FlatIndex::enqueue_range_route(QueryCtx &c, const CorpusView &v, CoarseKind kind, const CoarsePlan &cp, const RangeScratch &r,
                                    const void *d_q, size_t qpitch, uint32_t nq, const float *d_radii, const uint32_t *bm, uint32_t words,
                                    const RangeOut &out, cudaStream_t st, LaunchCounters &lc) {
    const uint32_t slots = cp.grid_x * cp.keep;
    CoarseOperands ops{};
    bool ok;
    if (kind == CoarseDirect8) {
        ok = cudaMemsetAsync(r.ovf, 0, nq * 4, st) == cudaSuccess;
        ok = ok && direct8_operands(d_q, qpitch, nq, reinterpret_cast<int32_t *>(r.qn2), st, lc, ops);
    } else if (kind == CoarseDirect16) {
        ok = launch_range_bound16(d_q, qpitch, nq, (uint32_t)dim_, dtype_, d_radii, shadow_max_norm_, r.thr, r.ovf, st) == cudaSuccess;
        ops = CoarseOperands{v.rows, v.pitch, d_q, qpitch, dtype_ == DT_BF16 ? 1 : 0, 0, nullptr, nullptr};
        lc.launches++;
    } else {
        ok = shadow_operands(d_q, qpitch, nq, r.q16, r.qn2, st, lc, ops);
        ok = ok && launch_range_bound(d_radii, nq, kCoarseEpsF16, r.qn2, shadow_max_norm_, (uint32_t)dim_, mkind_ == MT_L2 ? 1 : 0, r.thr, r.ovf,
                                      out.total, st) == cudaSuccess;
        lc.launches++;
    }
    cudaEventRecord(c.ev_start, st);
    ok = ok && launch_coarse(ops, v.n_rows, v.dim, nq, cp, r.cand, r.list_scratch, st, nullptr, kind == CoarseDirect8 ? d_radii : r.thr, r.ovf, bm,
                             words) == cudaSuccess;
    cudaEventRecord(c.ev_stop, st);
    lc.launches += 2;
    if (kind == CoarseDirect8)
        return ok && (out.flags ? launch_range_label_fold(r.cand, nq, slots, nullptr, r.ovf, d_id_to_label_, out.cap, out.hits, out.cnt, out.ok,
                                                          out.flags, st)
                                : launch_range_pack(r.cand, nq, slots, r.ovf, out.cap, out.hits, out.cnt, out.ok, st)) == cudaSuccess;
    if (!out.flags)
        return ok && launch_range_refine(v, d_q, qpitch, nq, slots, r.cand, d_radii, r.qn2, r.thr, r.ovf, out.hits, out.total, out.ok, out.cnt,
                                         out.off, st, out.cap) == cudaSuccess;
    // the kept rows stay at the front of each list segment (cap = slots onto cand itself: a copy onto itself)
    ok = ok && launch_range_refine(v, d_q, qpitch, nq, slots, r.cand, d_radii, r.qn2, r.thr, r.ovf, r.cand, out.total, out.ok, r.front, nullptr, st,
                                   slots) == cudaSuccess;
    lc.launches++;
    return ok && launch_range_label_fold(r.cand, nq, slots, r.front, nullptr, d_id_to_label_, out.cap, out.hits, out.cnt, out.ok, out.flags, st) ==
                     cudaSuccess;
}

// Enqueue on `st`: the `ke` best composites of each of `nq` device-resident stored-form queries into
// d_out [nq][ke].  Cosine fp32 batches take the tensor-core coarse pass + exact rescoring + proof, with
// the exact scan as an on-device fallback for unverified queries; everything else takes the exact
// fused scan.  ev_start/ev_stop of `c` bracket the dominant scan kernel.  A multi-value index selects labels instead
// (batch_scan_labels).
bool FlatIndex::batch_scan(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t ke, cudaStream_t st,
                           LaunchCounters &lc, uint64_t **d_result) {
    return multi_ ? batch_scan_labels(c, d_q, qpitch, nq, ke, st, lc, d_result) : batch_scan_rows(c, d_q, qpitch, nq, ke, st, lc, d_result);
}

// Row-tile stride of a sample pass that visits a fraction f = ke / (aim * row ranges) of the tiles, 1 % <= f <= 25 %: about `aim`
// slots per (query, row range) of the main pass then fall below the bound it yields.  Small corpora: at least tiles_per_k * ke
// tiles are visited, so that the sample still holds a few times k candidates.
static uint32_t sample_stride(const CoarsePlan &probe, uint32_t ke, double aim, double tiles_per_k) {
    const double f = std::min(0.25, std::max(0.01, (double)ke / (aim * probe.grid_x)));
    return (uint32_t)std::max(1.0, std::min(std::floor(1.0 / f), std::floor(probe.tiles / (tiles_per_k * ke))));
}

// The shadow copies run the first tier in two passes:
//   sample pass   every `stride`-th row tile, per (query, row range) the smallest approximate distance of 8 interleaved
//                 slices -> per query the bound T = (k-th smallest of its ranges x 8 minima) + 2 eps: k distinct rows
//                 lie at or below it, so it bounds the k-th best distance from above
//   main pass     all row tiles, every row with approximate distance < T is kept (fixed bound: no running thresholds,
//                 no list compaction, which a running threshold keeps the epilogue busy with)
// TF32 route: one pass with adaptive lists.  aim: the slots per (query, row range) of the main pass that should fall below the
// bound; filt: the main pass runs with row filters.
FlatIndex::KnnTiers FlatIndex::plan_knn_tiers(const CorpusView &v, uint32_t nq, CoarseKind kind, uint32_t ke, double aim, double tiles_per_k,
                                              bool filt) {
    KnnTiers t;
    const bool shadow = kind == CoarseF16 || kind == CoarseQ8;
    t.two_pass = shadow && coarse_fixed_enabled();
    t.tier2 = shadow && coarse_tier2_enabled();
    if (!t.two_pass) {
        t.main = plan_coarse(v, nq, kind, ke); // the adaptive lists ARE the first tier
    } else {
        t.main = plan_coarse(v, nq, kind, ke, 0, 1, 1, filt);
        // k in the hundreds: ranges x 32 slice minima barely hold k values.  The sample pass keeps adaptive lists of 128 per (query,
        // row range) instead; their union holds at least k distinct rows at or below its k-th smallest approximate distance, so
        // threshold_kernel's bound stands
        t.sample = ke > kCoarseMaxK ? plan_coarse(v, nq, kind, ke, kCoarseKeepWide, sample_stride(t.main, ke, aim, tiles_per_k), 0)
                                    : plan_coarse(v, nq, kind, ke, 0, sample_stride(t.main, ke, aim, tiles_per_k), 2);
    }
    // second tier: the queries whose first-tier proof failed (a list of the main pass overflowed: more than its capacity of rows of
    // one range within the bound — clustered corpora) are packed to the front and run once more with adaptive lists of 128 per row
    // range.  Nothing is known on the host: the tier's kernels read the count of open queries from device memory and leave at once
    // when it is zero.
    if (t.tier2) t.second = plan_coarse(v, nq, kind, ke, kCoarseKeepWide);
    return t;
}

void FlatIndex::KnnScratch::take(BatchScratch &s, const KnnTiers &t, uint32_t nq, size_t q_pitch, bool norms, bool q8) {
    cand = s.take<uint64_t>((size_t)nq * t.main.grid_x * t.main.keep);
    cand_s = s.take<uint64_t>(t.two_pass ? (size_t)nq * t.sample.grid_x * t.sample.keep : 0);
    cand_t2 = s.take<uint64_t>(t.tier2 ? (size_t)nq * t.second.grid_x * t.second.keep : 0);
    list_scratch = s.take<uint64_t>(std::max(std::max(t.main.scratch_elems, t.two_pass ? t.sample.scratch_elems : 0),
                                             t.tier2 ? t.second.scratch_elems : 0));
    q = s.take<uint8_t>(nq * q_pitch);
    q_t2 = s.take<uint8_t>(t.tier2 ? nq * q_pitch : 0);
    qn2 = s.take<float>(norms ? nq : 0); // |q|^2 per query
    qn2_t2 = s.take<float>(norms && t.tier2 ? nq : 0);
    qeps = s.take<float>(q8 ? nq : 0); // int8 copy: the error bound of each query
    qeps_t2 = s.take<float>(q8 && t.tier2 ? nq : 0);
    ok = s.take<uint32_t>(nq);
    idx = s.take<uint32_t>(nq);         // tier 2: indices of the open queries
    n2 = s.take<uint32_t>(nq ? 1 : 0);  //         and their count
    thr = s.take<float>(nq);            // fixed bound per query
    ovf = s.take<uint32_t>(nq);         // a list of the main pass ran full
    // entries of each list of the int8 copy's fixed pass, which publishes no padding
    cnt = s.take<uint32_t>(q8 && t.two_pass ? (size_t)nq * t.main.grid_x : 0);
}

bool FlatIndex::enqueue_knn_tiers(QueryCtx &c, const CorpusView &v, CoarseKind kind, const KnnTiers &t, const KnnScratch &s,
                                  const CoarseOperands &ops, const void *d_q32, size_t qpitch, uint32_t nq, uint32_t ke, uint64_t *out,
                                  const uint32_t *bm, uint32_t words, const uint64_t *row_label, cudaStream_t st, LaunchCounters &lc) {
    const float eps = coarse_eps(kind);
    bool ok = true;
    if (t.two_pass) {
        ok = launch_coarse(ops, v.n_rows, v.dim, nq, t.sample, s.cand_s, s.list_scratch, st, nullptr, nullptr, nullptr, bm, words) == cudaSuccess;
        ok = ok && launch_threshold(s.cand_s, nq, t.sample.grid_x, t.sample.keep, ke, eps, s.qn2, shadow_max_norm_, (uint32_t)dim_,
                                    mkind_ == MT_L2 ? 1 : 0, s.thr, s.ovf, st, s.qeps) == cudaSuccess;
        lc.launches += 2;
    }
    const float *thr = t.two_pass ? s.thr : nullptr;
    uint32_t *ovf = t.two_pass ? s.ovf : nullptr;
    cudaEventRecord(c.ev_start, st);
    ok = ok && launch_coarse(ops, v.n_rows, v.dim, nq, t.main, s.cand, s.list_scratch, st, nullptr, thr, ovf, bm, words, nullptr, s.cnt) ==
                   cudaSuccess;
    cudaEventRecord(c.ev_stop, st);
    // exact rescoring of the few candidates that can still matter + exact top-k + proof, one CTA per query
    ok = ok && launch_refine(v, d_q32, qpitch, nq, t.main.grid_x, t.main.keep, ke, s.cand, eps, s.qn2, shadow_max_norm_, s.ok, out, nullptr,
                             nullptr, st, thr, ovf, row_label, s.qeps, s.cnt) == cudaSuccess;
    lc.launches += 2;
    if (!t.tier2) return ok;
    ok = ok && launch_compact_unproven(s.ok, nq, s.idx, s.n2, st) == cudaSuccess;
    // the open queries' operand rows with their |q|^2 (fp16 copy) or error bound (int8 copy)
    ok = ok && launch_gather_queries(ops.queries, ops.qpitch, s.qeps ? s.qeps : s.qn2, s.idx, s.n2, nq, s.q_t2, s.qeps ? s.qeps_t2 : s.qn2_t2,
                                     st) == cudaSuccess;
    CoarseOperands ops2 = ops;
    ops2.queries = s.q_t2;
    if (ops.q_norm2) ops2.q_norm2 = s.qn2_t2;
    ok = ok && launch_coarse(ops2, v.n_rows, v.dim, nq, t.second, s.cand_t2, s.list_scratch, st, s.n2, nullptr, nullptr, bm, words,
                             bm ? s.idx : nullptr) == cudaSuccess;
    ok = ok && launch_refine(v, d_q32, qpitch, nq, t.second.grid_x, t.second.keep, ke, s.cand_t2, eps, s.qn2_t2, shadow_max_norm_, s.ok, out,
                             s.idx, s.n2, st, nullptr, nullptr, row_label, s.qeps_t2) == cudaSuccess;
    lc.launches += 4;
    return ok;
}

bool FlatIndex::batch_scan_rows(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t ke, cudaStream_t st,
                                LaunchCounters &lc, uint64_t **d_result, bool tc_only) {
    const CorpusView v = view();
    const ScanPlan sp = plan_scan_topk(v, nq, ke);
    const int cmode = coarse_mode();
    // fp16 / bf16 corpora: the tensor-core GEMM with fp32 accumulation IS the distance (within the 1e-2 bar by four
    // orders of magnitude), so the batch is one kernel + the usual final selection — no shadow, no rescoring
    const bool is16 = dtype_ == DT_F16 || dtype_ == DT_BF16, is8 = dtype_ == DT_I8 || dtype_ == DT_U8;
    const CoarseKind dkind = is16 ? CoarseDirect16 : CoarseDirect8;
    // int8 / uint8 L2: the int32 |row|^2 table is brought up to date on `st` first (no HBM for it: the exact scan)
    if (cmode != 0 && nq >= 16 && (is16 || is8) && coarse_supported(v, nq, ke, dkind) && (!int_l2() || ensure_shadow(st))) {
        const CoarseOperands ops16{v.rows, v.pitch, d_q, qpitch, dtype_ == DT_BF16 ? 1 : 0, mkind_ == MT_COS ? 1 : 0, nullptr, nullptr};
        last_batch_coarse_ = true;
        last_batch_path_ = 2;
        c.d_last_ok = nullptr;
        c.last_ok_n = 0;
        const CoarsePlan cp = plan_coarse(v, nq, dkind, ke);
        // 16-bit corpora: the fixed-bound scheme of the fp32 route without the error term — the GEMM result IS the distance, so
        // T = the k-th smallest slice minimum of the sample pass bounds the k-th best distance from above and the main pass
        // keeps every row with d <= T (no running thresholds, no compaction); a list that runs full sends the query to the
        // adaptive kernel.  (int8 distances are small integers with massive ties: they stay on the adaptive lists.)
        const CoarsePlan probe = plan_coarse(v, nq, dkind, ke, 0, 1, 1);
        if (is16 && probe.mode == 1 && coarse_fixed_enabled()) {
            // aim at 64 of the 256 slots per (query, row range); the sample holds a few times k slice minima (4 per visited tile)
            const CoarsePlan cps = plan_coarse(v, nq, dkind, ke, 0, sample_stride(probe, ke, 64.0, 2.0), 2);
            const bool tier2 = coarse_tier2_enabled();
            const size_t nO = (size_t)nq * ke;
            const size_t scratch = std::max(std::max(probe.scratch_elems, cps.scratch_elems), tier2 ? cp.scratch_elems : 0);
            uint64_t *cand_m, *cand_s, *cand_t2, *out2, *list_scratch;
            uint8_t *q_t2;
            uint32_t *d_ok, *d_idx, *d_n2, *d_ovf;
            float *d_thr;
            const auto layout = [&](void *base) {
                BatchScratch s(base);
                cand_m = s.take<uint64_t>((size_t)nq * probe.grid_x * probe.keep);
                cand_s = s.take<uint64_t>((size_t)nq * cps.grid_x * cps.keep);
                cand_t2 = s.take<uint64_t>(tier2 ? (size_t)nq * cp.grid_x * cp.keep : 0);
                out2 = s.take<uint64_t>(nO);
                list_scratch = s.take<uint64_t>(scratch);
                q_t2 = s.take<uint8_t>(tier2 ? (size_t)nq * qpitch : 0); // tier 2: the open queries, packed to the front
                d_ok = s.take<uint32_t>(nq);
                d_idx = s.take<uint32_t>(nq); // tier 2: indices of the open queries
                d_n2 = s.take<uint32_t>(1);   //         and their count
                d_thr = s.take<float>(nq);    // fixed bound per query
                d_ovf = s.take<uint32_t>(nq); // a list of the main pass ran full
                return s.words();
            };
            if (!c.need_cand(layout(nullptr)) || !c.need_out(nO)) return false;
            layout(c.d_cand);
            c.d_last_ok = d_ok;
            c.last_ok_n = nq;
            bool ok = launch_coarse(ops16, v.n_rows, v.dim, nq, cps, cand_s, list_scratch, st) == cudaSuccess;
            ok = ok && launch_threshold(cand_s, nq, cps.grid_x, cps.keep, ke, 0.0f, nullptr, 0.0f, (uint32_t)dim_, 0, d_thr, d_ovf, st) == cudaSuccess;
            cudaEventRecord(c.ev_start, st);
            ok = ok && launch_coarse(ops16, v.n_rows, v.dim, nq, probe, cand_m, list_scratch, st, nullptr, d_thr, d_ovf) == cudaSuccess;
            cudaEventRecord(c.ev_stop, st);
            ok = ok && launch_final_select(cand_m, nq, (uint32_t)(probe.grid_x * probe.keep), ke, c.d_out, st, &lc) == cudaSuccess;
            ok = ok && launch_flags_from_overflow(d_ovf, nq, d_ok, st) == cudaSuccess;
            lc.launches += 4;
            if (tier2) {
                ok = ok && launch_compact_unproven(d_ok, nq, d_idx, d_n2, st) == cudaSuccess;
                ok = ok && launch_gather_queries(d_q, qpitch, nullptr, d_idx, d_n2, nq, q_t2, nullptr, st) == cudaSuccess;
                CoarseOperands ops2 = ops16;
                ops2.queries = q_t2;
                ok = ok && launch_coarse(ops2, v.n_rows, v.dim, nq, cp, cand_t2, list_scratch, st, d_n2) == cudaSuccess;
                ok = ok && launch_final_select(cand_t2, nq, (uint32_t)(cp.grid_x * cp.keep), ke, out2, st, &lc, d_n2) == cudaSuccess;
                ok = ok && launch_scatter_rows(out2, d_idx, d_n2, nq, ke, c.d_out, d_ok, st) == cudaSuccess;
                lc.launches += 4;
            }
            coarse_batches_++;
            *d_result = c.d_out;
            return ok;
        }
        uint64_t *cand, *list_scratch;
        int32_t *d_qn;
        const auto layout = [&](void *base) {
            BatchScratch s(base);
            cand = s.take<uint64_t>((size_t)nq * cp.grid_x * cp.keep);
            list_scratch = s.take<uint64_t>(cp.scratch_elems);
            d_qn = s.take<int32_t>(int_l2() ? nq : 0); // int8 / uint8 L2: |q|^2 per query
            return s.words();
        };
        if (!c.need_cand(layout(nullptr)) || !c.need_out((size_t)nq * ke)) return false;
        layout(c.d_cand);
        CoarseOperands ops = ops16;
        bool ok = !is8 || direct8_operands(d_q, qpitch, nq, d_qn, st, lc, ops);
        cudaEventRecord(c.ev_start, st);
        ok = ok && launch_coarse(ops, v.n_rows, v.dim, nq, cp, cand, list_scratch, st) == cudaSuccess;
        cudaEventRecord(c.ev_stop, st);
        ok = ok && launch_final_select(cand, nq, (uint32_t)(cp.grid_x * cp.keep), ke, c.d_out, st, &lc) == cudaSuccess;
        lc.launches++;
        coarse_batches_++;
        *d_result = c.d_out;
        return ok;
    }
    CoarseKind kind = cmode == 2 ? CoarseTF32 : CoarseF16;
    // cosine: unit vectors, constant error bound, either operand kind.  L2 / raw inner product (fp32): the fp16 route only,
    // error bound from the row and query norms
    const bool unit = unit_rows();
    // k > kCoarseMaxK (DESIGN.md §4.5): the fp16 route's two-pass first tier, for batches of 16 queries and more
    const bool wide = ke > kCoarseMaxK;
    const bool eligible = cmode != 0 && !coarse_disabled_ && dtype_ == DT_F32 && (unit || cmode == 1) &&
                          (nq >= 16 || (!wide && single_query_takes_coarse(ke, nullptr, q8_route(nq, ke)))) && (!wide || coarse_fixed_enabled());
    // unit rows with k <= kCoarseMaxK: the int8 copy (DESIGN.md §4.2), unless its bounds are not finite (a NaN or inf row)
    if (eligible && kind == CoarseF16 && q8_route(nq, ke) && ensure_shadow(st, true) && std::isfinite(shadow8_delta_) &&
        std::isfinite(shadow8_xmax_))
        kind = CoarseQ8;
    bool coarse = eligible && coarse_supported(v, nq, ke, kind);
    if (eligible && kind == CoarseF16 && (!coarse || !ensure_shadow(st))) { // rows too wide for the 16-bit kernel's shared memory, or no HBM for the shadow
        kind = CoarseTF32;
        coarse = unit && coarse_supported(v, nq, ke, kind);
    }
    if (coarse && !shadow_values_in_range()) coarse = false;
    last_batch_coarse_ = coarse;
    last_batch_path_ = coarse ? 1 : 0;
    last_shadow_bits_ = !coarse ? 0 : kind == CoarseQ8 ? 8 : kind == CoarseF16 ? 16 : 0;
    if (!coarse && tc_only) {
        *d_result = nullptr;
        return true;
    }
    // the exact top-k of k > kMaxFusedK: whole batches no route serves here, the queries the route leaves open below
    const WidePlan wp = wide ? plan_topk_wide(v.n_rows, nq) : WidePlan{};
    if (!coarse && wide) {
        if (!c.need_scores(wp.score_elems) || !c.need_cand(wp.cand_elems) || !c.need_out((size_t)nq * ke)) return false;
        cudaEventRecord(c.ev_start, st);
        const bool ok = launch_topk_wide(v, d_q, qpitch, nq, ke, nullptr, nullptr, wp, c.d_scores, c.d_cand, c.d_out, c.d_abort, st, &lc) ==
                        cudaSuccess;
        cudaEventRecord(c.ev_stop, st);
        *d_result = c.d_out;
        return ok;
    }
    if (!coarse) {
        if (!c.need_cand(sp.cand_elems) || !c.need_out((size_t)nq * ke)) return false;
        cudaEventRecord(c.ev_start, st);
        bool ok = launch_scan_topk(v, d_q, qpitch, nq, ke, sp, c.d_cand, st, &lc, nullptr, c.d_abort) == cudaSuccess;
        cudaEventRecord(c.ev_stop, st);
        ok = ok && launch_final_select(c.d_cand, nq, sp.lists_per_query * ke, ke, c.d_out, st, &lc) == cudaSuccess;
        *d_result = c.d_out;
        return ok;
    }
    const bool q8 = kind == CoarseQ8, shadow = kind == CoarseF16 || q8;
    // expected rows below T per (query, row range) = k / (sample fraction * ranges): aim at 24 of the 96 slots; the sample holds a
    // few times k slice minima (4 per visited tile).  The int8 copy's bound is about 7x the fp16 one's, and the rows within 2 eps
    // of the k-th distance, not k / f, fill most of its lists of 256: it samples about 4 % at k = 10 over 30 ranges (aim 8), which
    // keeps the rows below the bound near a quarter of a list on uniform unit rows.  k in the hundreds: aim at 128 of the 256
    // slots of the main pass; the sample holds about 4 k rows (128 per visited tile).
    const KnnTiers t = plan_knn_tiers(v, nq, kind, ke, wide ? 128.0 : q8 ? 8.0 : 24.0, wide ? 1 / 32.0 : 2.0, false);
    const size_t nO = (size_t)nq * ke;
    // the queries in the operand type of the copy: fp16 rows, or int8 rows with their scale (coarse_q8_pitch)
    const size_t q_pitch = !shadow ? 0 : q8 ? coarse_q8_pitch((uint32_t)dim_) : f16_query_pitch();
    const size_t nO12 = wide ? 0 : nO; // k > kMaxFusedK: the tiers write the answer rows in place, no out1 / out2
    KnnScratch ks;
    uint64_t *out1, *out2, *cand2;
    const auto layout = [&](void *base) {
        BatchScratch s(base);
        ks.take(s, t, nq, q_pitch, !unit, q8);
        out1 = s.take<uint64_t>(nO12);
        out2 = s.take<uint64_t>(nO12);
        // k > kMaxFusedK: the exact fallback's chunk-select lists take the place of the fused scan's
        cand2 = s.take<uint64_t>(wide ? wp.cand_elems : sp.cand_elems);
        return s.words();
    };
    if (!c.need_cand(layout(nullptr)) || !c.need_out(nO) || (wide && !c.need_scores(wp.score_elems))) return false;
    layout(c.d_cand);
    if (wide) out1 = c.d_out; // both tiers and the exact fallback write their rows of the answer in place (no blend)
    c.d_last_ok = ks.ok;
    c.last_ok_n = nq;
    CoarseOperands ops{v.rows, v.pitch, d_q, qpitch, 0, 0, nullptr, nullptr};
    bool ok = true;
    if (kind == CoarseF16) {
        ok = shadow_operands(d_q, qpitch, nq, ks.q, ks.qn2, st, lc, ops);
    } else if (q8) {
        ok = launch_quantize_queries(d_q, qpitch, (uint32_t)dim_, nq, ks.q, ks.qeps, shadow8_delta_, shadow8_xmax_, st) == cudaSuccess;
        ops = CoarseOperands{d_shadow8_, 0, ks.q, q_pitch, 1, 0, d_tscale_, nullptr};
        lc.launches++;
    }
    ok = ok && enqueue_knn_tiers(c, v, kind, t, ks, ops, d_q, qpitch, nq, ke, out1, nullptr, 0, nullptr, st, lc);
    if (wide) {
        // exact fallback of the open queries, entirely on device; with none open, every launch exits at once
        ok = ok && launch_compact_unproven(ks.ok, nq, ks.idx, ks.n2, st) == cudaSuccess;
        ok = ok && launch_topk_wide(v, d_q, qpitch, nq, ke, ks.idx, ks.n2, wp, c.d_scores, cand2, c.d_out, c.d_abort, st, &lc) == cudaSuccess;
        lc.launches++;
        coarse_batches_++;
        *d_result = c.d_out;
        return ok;
    }
    // exact fallback, entirely on device: CTAs whose queries are all verified exit at once
    ok = ok && launch_scan_topk(v, d_q, qpitch, nq, ke, sp, cand2, st, &lc, ks.ok, c.d_abort) == cudaSuccess;
    ok = ok && launch_final_select(cand2, nq, sp.lists_per_query * ke, ke, out2, st, &lc) == cudaSuccess;
    ok = ok && launch_blend(ks.ok, out1, out2, nq, ke, c.d_out, st, &lc) == cudaSuccess;
    coarse_batches_++;
    *d_result = c.d_out;
    return ok;
}

// Multi-value index (DESIGN.md §4.4).  Rows are ordered by (score, row id) and a label by its best row.  If a tensor-core route
// applies, it selects the K = min(128, kl * m, n) best rows of each query (m = most rows any label owns) and label_select takes
// their first kl distinct labels; that is exact when the K rows hold kl distinct labels, which K >= kl * m guarantees unless
// K was capped at 128.  Queries with fewer labels, and whole batches no tensor-core route serves, run the label-aware exact
// scan.  Nothing returns to the host in between.
// host_fallback (the host API): the label-aware exact scan runs only for corpora too small for the tensor-core routes.  Elsewhere
// it is slower than one query at a time (DESIGN.md §4.4), so the caller answers those queries with topk(): the ones whose
// c.d_last_ok flag is 3 after a row route, or all of them when *d_result comes back NULL.
bool FlatIndex::batch_scan_labels(QueryCtx &c, const void *d_q, size_t qpitch, uint32_t nq, uint32_t kl, cudaStream_t st, LaunchCounters &lc,
                                  uint64_t **d_result, bool host_fallback) {
    const CorpusView v = view();
    const uint32_t K = (uint32_t)std::min<size_t>(std::min<size_t>(kMaxFusedK, (size_t)kl * max_rows_per_label()), v.n_rows);
    const ScanPlan sp = plan_scan_topk(v, nq, kl, true);
    const size_t nO = (size_t)nq * kl;
    uint64_t *out1, *out2, *cand;
    uint32_t *lab_ok, *flags;
    const auto layout = [&](void *base) {
        BatchScratch s(base);
        out1 = s.take<uint64_t>(nO);              // label answers
        out2 = s.take<uint64_t>(nO);              // exact answers
        cand = s.take<uint64_t>(sp.cand_elems);   // lists of the exact scan
        lab_ok = s.take<uint32_t>(nq);            // label check per query
        flags = s.take<uint32_t>(nq);             // reported flags
        return s.words();
    };
    // d_lab, not d_cand: the row stage below lays out its own scratch there
    if (!c.need_lab(layout(nullptr))) return false;
    layout(c.d_lab);
    uint64_t *rows = nullptr;
    if (!batch_scan_rows(c, d_q, qpitch, nq, K, st, lc, &rows, true)) return false;
    bool ok = true;
    if (rows) {
        // rows: [nq][K] in c.d_out; the label answers are blended back into it
        ok = launch_label_select(rows, nq, K, d_id_to_label_, kl, c.d_last_ok, out1, lab_ok, flags, st, &lc) == cudaSuccess;
        c.d_last_ok = flags;
        c.last_ok_n = nq;
        if (host_fallback) {
            ok = ok && cudaMemcpyAsync(c.d_out, out1, nO * 8, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
        } else {
            ok = ok && launch_scan_topk(v, d_q, qpitch, nq, kl, sp, cand, st, &lc, lab_ok, c.d_abort, d_id_to_label_) == cudaSuccess;
            ok = ok && launch_final_select_labels(cand, nq, sp.lists_per_query * kl, kl, d_id_to_label_, out2, st, &lc) == cudaSuccess;
            ok = ok && launch_blend(lab_ok, out1, out2, nq, kl, c.d_out, st, &lc) == cudaSuccess;
            cudaEventRecord(c.ev_stop, st); // the timed span runs from the row stage's main pass through the label-aware scan
        }
    } else if (host_fallback && v.n_rows >= 65536) {
        c.d_last_ok = nullptr;
        *d_result = nullptr;
        return true;
    } else {
        c.d_last_ok = nullptr;
        if (!c.need_out(nO)) return false;
        cudaEventRecord(c.ev_start, st);
        ok = launch_scan_topk(v, d_q, qpitch, nq, kl, sp, cand, st, &lc, nullptr, c.d_abort, d_id_to_label_) == cudaSuccess;
        cudaEventRecord(c.ev_stop, st);
        ok = ok && launch_final_select_labels(cand, nq, sp.lists_per_query * kl, kl, d_id_to_label_, c.d_out, st, &lc) == cudaSuccess;
    }
    *d_result = c.d_out;
    return ok;
}

int FlatIndex::topk_batch(const void *qs, size_t qstride, size_t nq, size_t k, VecSimQueryParams *qp, size_t *out_labels,
                          double *out_scores) {
    void *tctx = qp ? qp->timeoutCtx : nullptr;
    last_mode_ = STANDARD_KNN;
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (size_t i = 0; i < nq * k; i++) {
        out_labels[i] = SIZE_MAX;
        out_scores[i] = nan;
    }
    if (nq == 0 || k == 0) return VecSim_QueryReply_OK;
    if (!flush()) return -1;
    const size_t n = count_;
    if (n == 0) return VecSim_QueryReply_OK;
    if (timed_out(tctx)) return VecSim_QueryReply_TimedOut;
    const auto one_query = [&](size_t i) { // the generic path for query i
        VecSimQueryReply *r = topk(static_cast<const uint8_t *>(qs) + i * qstride, k, qp, BY_SCORE);
        const int code = r->code;
        for (size_t j = 0; j < k; j++) {
            out_labels[i * k + j] = j < r->results.size() ? r->results[j].id : SIZE_MAX;
            out_scores[i * k + j] = j < r->results.size() ? r->results[j].score : nan;
        }
        delete r;
        return code;
    };
    // single-value, kMaxFusedK < min(k, n) <= kMaxWideK: batches the fp32 route serves run as one batch (DESIGN.md §4.5)
    const bool wide = !multi_ && std::min(k, n) > (size_t)kMaxFusedK && std::min(k, n) <= (size_t)kMaxWideK;
    if (multi_ ? k > (size_t)kMaxFusedK : (std::min(k, n) > (size_t)kMaxFusedK && !wide)) { // generic path, one query at a time
        for (size_t i = 0; i < nq; i++) {
            const int code = one_query(i);
            if (code != VecSim_QueryReply_OK) return code;
        }
        return VecSim_QueryReply_OK;
    }
    if (multi_ && !sync_labels_to_device()) return -1;
    auto c = checkout();
    if (!c) return -1;
    const size_t qpitch = query_pitch();
    const uint32_t ke = (uint32_t)std::min(k, multi_ ? label_count() : n); // a multi-value index answers labels
    LaunchCounters lc;
    bool ok = stage_queries(*c, qs, qstride, nq, true);
    uint64_t *d_res = nullptr;
    // multi-value: queries the label stage could not prove, or all of them, are answered one at a time below (batch_scan_labels)
    bool per_query_all = false;
    const uint32_t *d_flags = nullptr;
    if (multi_) {
        ok = ok && c->need_ids(nq) && batch_scan_labels(*c, c->d_query, qpitch, (uint32_t)nq, ke, c->stream, lc, &d_res, true);
        per_query_all = ok && !d_res;
        d_flags = c->d_last_ok;
        ok = ok && (!d_flags || cudaMemcpyAsync(c->h_ids, d_flags, nq * 4, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess);
    } else if (wide) {
        // no route for this batch: the host API keeps answering it one query at a time (d_res comes back NULL)
        ok = ok && batch_scan_rows(*c, c->d_query, qpitch, (uint32_t)nq, ke, c->stream, lc, &d_res, true);
        per_query_all = ok && !d_res;
    } else {
        ok = ok && batch_scan(*c, c->d_query, qpitch, (uint32_t)nq, ke, c->stream, lc, &d_res);
    }
    ok = ok && (per_query_all || cudaMemcpyAsync(c->h_out, c->d_out, nq * ke * 8, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess);
    launches_total_ += lc.launches;
    if (ok) {
        const int w = wait_or_abandon(*c, tctx); // a full exact-scan fallback no longer holds a timed-out caller
        if (w == 1) {
            checkin(std::move(c));
            return VecSim_QueryReply_TimedOut;
        }
        ok = w == 0;
    }
    if (per_query_all && ok) { // the stream is idle: wait_polling above saw the query upload finish
        checkin(std::move(c));
        for (size_t i = 0; i < nq; i++) {
            const int code = one_query(i);
            if (code != VecSim_QueryReply_OK) return code;
        }
        return VecSim_QueryReply_OK;
    }
    std::vector<size_t> open; // multi-value queries whose label check failed (flag 3)
    if (ok) {
        record_scan(c.get(), (uint64_t)n * stored_bytes_);
        if (d_flags)
            for (size_t i = 0; i < nq; i++)
                if (c->h_ids[i] == 3u) open.push_back(i);
        VecSimQueryReply rr;
        for (size_t i = 0; i < nq; i++) {
            rr.results.clear();
            for (uint32_t j = 0; j < ke && c->h_out[i * ke + j] != kEmptySlot; j++)
                rr.results.push_back(decode(c->h_out[i * ke + j], id_to_label_));
            finish_reply(&rr, BY_SCORE);
            for (size_t j = 0; j < rr.results.size(); j++) {
                out_labels[i * k + j] = rr.results[j].id;
                out_scores[i * k + j] = rr.results[j].score;
            }
        }
    }
    checkin(std::move(c));
    if (!ok) return -1;
    const int path = last_batch_path_; // LastBatchPath reports the batch's row stage, not the per-query answers below
    for (size_t i : open) {
        const int code = one_query(i);
        if (code != VecSim_QueryReply_OK) {
            last_batch_path_ = path;
            return code;
        }
    }
    last_batch_path_ = path;
    if (timed_out(tctx)) return VecSim_QueryReply_TimedOut;
    return VecSim_QueryReply_OK;
}

int FlatIndex::topk_batch_device(const void *d_q, size_t nq, size_t k, int64_t *d_labels, float *d_scores, cudaStream_t s) {
    if (nq == 0 || k == 0) return 0;
    if (!flush() || !sync_labels_to_device()) return -1;
    const size_t n = count_;
    if (k > (size_t)(multi_ ? kMaxFusedK : kMaxWideK)) return -1; // single-value, k > kMaxFusedK: DESIGN.md §4.5
    // Scratch of this entry point is stream-ordered: one dedicated context, reused call after call.
    // Callers enqueue on one stream (or synchronise between streams), as with any async API.
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_) dev_ctx_ = checkout();
    QueryCtx *c = dev_ctx_.get();
    if (!c) return -1;
    collect_dev_timing_locked(); // the previous call's scan events (stream-ordered before this call)
    const size_t qpitch = query_pitch();
    const uint32_t ke = (uint32_t)std::min(k, std::max<size_t>(multi_ ? label_count() : n, 1));
    cudaStream_t st = s ? s : cudaStreamLegacy; // NULL = the legacy default stream, as everywhere in CUDA
    LaunchCounters lc;
    bool ok = true;
    if (n == 0) {
        ok = cudaMemsetAsync(d_labels, 0xFF, nq * k * 8, st) == cudaSuccess;
    } else {
        uint64_t *d_res = nullptr;
        ok = c->need_out(nq * k);
        if (!ok) {
        } else if (ke == k) {
            ok = batch_scan(*c, d_q, qpitch, (uint32_t)nq, ke, st, lc, &d_res);
        } else {
            // fewer rows than k: select [nq][ke], then widen the rows to [nq][k] (tail = empty)
            ok = batch_scan(*c, d_q, qpitch, (uint32_t)nq, ke, st, lc, &d_res);
            ok = ok && c->need_ids(nq * k * 2);
            uint64_t *wide = reinterpret_cast<uint64_t *>(c->d_ids);
            ok = ok && cudaMemsetAsync(wide, 0xFF, nq * k * 8, st) == cudaSuccess;
            ok = ok && cudaMemcpy2DAsync(wide, k * 8, d_res, ke * 8, ke * 8, nq, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(c->d_out, wide, nq * k * 8, cudaMemcpyDeviceToDevice, st) == cudaSuccess;
        }
        ok = ok && launch_unpack_results(c->d_out, (uint32_t)nq, (uint32_t)k, d_id_to_label_, d_labels, d_scores, st, &lc) == cudaSuccess;
        dev_timing_pending_ = ok;
        dev_timing_bytes_ = (uint64_t)n * stored_bytes_;
    }
    launches_total_ += lc.launches;
    return ok ? 0 : -1;
}

VecSimQueryReply *FlatIndex::range(const void *q, double radius, VecSimQueryParams *qp, VecSimQueryReply_Order order) {
    auto *rep = new VecSimQueryReply();
    last_mode_ = RANGE_QUERY;
    void *tctx = qp ? qp->timeoutCtx : nullptr;
    if (!flush()) return rep;
    const size_t n = count_;
    if (n == 0) return rep;
    if (timed_out(tctx)) {
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    auto c = checkout();
    if (!c) return rep;
    LaunchCounters lc;
    bool ok = c->need_scores(n) && c->need_cand(n) && stage_queries(*c, q, 0, 1, true);
    const CorpusView v = view();
    ok = ok && launch_scan_scores(v, c->d_query, c->d_scores, c->stream, &lc) == cudaSuccess;
    ok = ok && launch_range_compact(c->d_scores, (uint32_t)n, (float)radius, c->d_cand, c->d_count, c->stream, &lc) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(c->h_count, c->d_count, 4, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c->stream) == cudaSuccess;
    if (ok) {
        const uint32_t m = *c->h_count;
        ok = c->need_out(m);
        ok = ok && cudaMemcpyAsync(c->h_out, c->d_cand, (size_t)m * 8, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess;
        ok = ok && cudaStreamSynchronize(c->stream) == cudaSuccess;
        if (ok) {
            if (multi_) { // best score per label (brute_force_multi.h range container)
                std::unordered_map<size_t, uint32_t> best;
                for (uint32_t i = 0; i < m; i++) {
                    const uint64_t comp = c->h_out[i];
                    const size_t label = id_to_label_[(uint32_t)comp];
                    const uint32_t key = (uint32_t)(comp >> 32);
                    auto it = best.find(label);
                    if (it == best.end() || key < it->second) best[label] = key;
                }
                for (auto &kv : best) rep->results.push_back({kv.first, (double)key_to_float(kv.second)});
            } else {
                rep->results.reserve(m);
                for (uint32_t i = 0; i < m; i++) rep->results.push_back(decode(c->h_out[i], id_to_label_));
            }
        }
    }
    launches_total_ += lc.launches;
    checkin(std::move(c));
    if (!ok) rep->results.clear();
    if (timed_out(tctx)) rep->code = VecSim_QueryReply_TimedOut; // brute_force.h:306-309 keeps partial results
    finish_reply(rep, order);
    return rep;
}

// Range batches (DESIGN.md §4, "Range queries"): an eligible fp32 batch takes ONE fixed-bound main pass over the fp16 shadow
// with the bound radius + eps per query, exact rescoring of the kept rows and a per-query proof; every other batch, and every
// query whose proof fails, is answered by range() one query at a time.
int FlatIndex::range_batch(const void *qs, size_t qstride, size_t nq, const double *radii, VecSimQueryParams *qp, VecSimQueryReply_Order order,
                           VecSimQueryReply **replies, uint32_t *out_flags) {
    void *tctx = qp ? qp->timeoutCtx : nullptr;
    last_mode_ = RANGE_QUERY;
    for (size_t i = 0; i < nq; i++) {
        replies[i] = nullptr;
        if (out_flags) out_flags[i] = 0;
    }
    if (nq == 0) return VecSim_QueryReply_OK;
    const auto all_timed_out = [&]() {
        for (size_t i = 0; i < nq; i++) {
            if (!replies[i]) replies[i] = new VecSimQueryReply();
            replies[i]->results.clear();
            replies[i]->code = VecSim_QueryReply_TimedOut;
        }
        return (int)VecSim_QueryReply_TimedOut;
    };
    if (timed_out(tctx)) return all_timed_out();
    if (!flush()) return -1;
    const size_t n = count_;
    const CorpusView v = view();
    // k plays no part in a range query: any k the planner accepts
    bool route = n > 0 && nq <= 0xFFFFFFFFu && coarse_mode() == 1 && dtype_ == DT_F32 && !multi_ && !coarse_disabled_ && coarse_fixed_enabled() &&
                 coarse_supported(v, (uint32_t)nq, 1, CoarseF16) && (nq >= 16 || single_query_takes_coarse(1));
    std::unique_ptr<QueryCtx> c;
    if (route) {
        c = checkout();
        route = c && ensure_shadow(c->stream);
    }
    if (route && !shadow_values_in_range()) route = false;
    if (route) {
        const uint32_t nq32 = (uint32_t)nq;
        cudaStream_t st = c->stream;
        LaunchCounters lc;
        // stored-form queries, then the radii as float (the reference compares score <= DistType(radius))
        const size_t qpitch = query_pitch();
        const std::vector<float> radii_f(radii, radii + nq);
        bool ok = stage_queries(*c, qs, qstride, nq, true, radii_f.data(), nq * sizeof(float));
        const float *d_radius = reinterpret_cast<const float *>(c->d_query + qpitch * nq);
        const CoarsePlan cp = plan_coarse(v, nq32, CoarseF16, 1, 0, 1, 1);
        const size_t slots = (size_t)cp.grid_x * cp.keep;
        RangeScratch rs;
        uint64_t *hits;
        uint32_t *d_res;
        const auto layout = [&](void *base) {
            BatchScratch s(base);
            rs.take(s, *this, CoarseF16, cp, nq32, false);
            hits = s.take<uint64_t>(nq * slots);
            d_res = s.take<uint32_t>(3 * nq + 1); // [ok nq][count nq][offset nq][hits in total]
            return s.words();
        };
        ok = ok && c->need_cand(layout(nullptr)) && c->need_ids(3 * nq + 1);
        layout(c->d_cand);
        ok = ok && enqueue_range_route(*c, v, CoarseF16, cp, rs, c->d_query, qpitch, nq32, d_radius, nullptr, 0,
                                       RangeOut{hits, 0, d_res, d_res + nq, d_res + 2 * nq, d_res + 3 * nq, nullptr}, st, lc);
        ok = ok && cudaMemcpyAsync(c->h_ids, d_res, (3 * nq + 1) * sizeof(uint32_t), cudaMemcpyDeviceToHost, st) == cudaSuccess;
        launches_total_ += lc.launches;
        coarse_batches_++;
        if (ok) {
            const int w = wait_or_abandon(*c, tctx);
            if (w == 1) { // deadline passed while the pass was running
                checkin(std::move(c));
                return all_timed_out();
            }
            ok = w == 0;
        }
        const uint32_t *h_ok = c->h_ids, *h_cnt = h_ok + nq, *h_off = h_cnt + nq;
        if (ok) {
            record_scan(c.get(), (uint64_t)n * stored_bytes_);
            const uint32_t total = h_ok[3 * nq]; // only the occupied part of the result buffer crosses PCIe
            ok = c->need_out(total) && cudaMemcpyAsync(c->h_out, hits, (size_t)total * 8, cudaMemcpyDeviceToHost, st) == cudaSuccess &&
                 cudaStreamSynchronize(st) == cudaSuccess;
        }
        if (ok) {
            for (size_t i = 0; i < nq; i++) {
                if (!h_ok[i]) continue;
                auto *rep = new VecSimQueryReply();
                rep->results.reserve(h_cnt[i]);
                for (uint32_t j = 0; j < h_cnt[i]; j++) rep->results.push_back(decode(c->h_out[(size_t)h_off[i] + j], id_to_label_));
                finish_reply(rep, order);
                replies[i] = rep;
                if (out_flags) out_flags[i] = 1;
            }
        }
        checkin(std::move(c));
        if (!ok) {
            log("warning", "vecsim_b200: range batch failed on device");
            for (size_t i = 0; i < nq; i++) {
                delete replies[i];
                replies[i] = nullptr;
                if (out_flags) out_flags[i] = 0;
            }
            return -1;
        }
    } else if (c) {
        checkin(std::move(c));
    }
    // queries the route did not answer (or the whole batch): one exact scan each
    for (size_t i = 0; i < nq; i++)
        if (!replies[i]) replies[i] = range(static_cast<const uint8_t *>(qs) + i * qstride, radii[i], qp, order);
    last_mode_ = RANGE_QUERY;
    const bool late = timed_out(tctx); // as range(): the replies keep what was found
    int rc = VecSim_QueryReply_OK;
    for (size_t i = 0; i < nq; i++) {
        if (late) replies[i]->code = VecSim_QueryReply_TimedOut;
        if (replies[i]->code == VecSim_QueryReply_TimedOut) rc = VecSim_QueryReply_TimedOut;
    }
    return rc;
}

int FlatIndex::range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_labels,
                                  float *d_scores, uint32_t *d_counts, cudaStream_t s) {
    if (multi_) return -1;
    return range_device(d_q, nq, d_radii, cap, order, d_labels, d_scores, d_counts, s);
}

int FlatIndex::label_range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order,
                                        int64_t *d_labels, float *d_scores, uint32_t *d_counts, cudaStream_t s) {
    if (!multi_) return range_batch_device(d_q, nq, d_radii, cap, order, d_labels, d_scores, d_counts, s);
    return range_device(d_q, nq, d_radii, cap, order, d_labels, d_scores, d_counts, s);
}

// Device range batches (DESIGN.md §4.11): one route per batch, then the exact scan on the device for the queries it left open
// (or for the whole batch), then one CTA per query orders its hits and maps rows to labels.  Hits are gathered as composites in
// d_labels itself ([nq][cap] uint64) with the true count in d_counts.  Nothing waits on the host except ensure_shadow (and, on a
// multi-value index, the label tables' rebuild after a mutation).  Multi-value index (§4.12): a route's proven row answer is folded
// to one entry per label (launch_range_label_fold) and the exact scan folds label-major over the CSR label table.
int FlatIndex::range_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order, int64_t *d_labels,
                            float *d_scores, uint32_t *d_counts, cudaStream_t s) {
    if (cap == 0 || cap > kRangeDeviceMaxCap || (order != BY_ID && order != BY_SCORE) || nq > 0xFFFFFFFFu) return -1;
    last_mode_ = RANGE_QUERY;
    if (nq == 0) return 0;
    if (!flush() || !sync_labels_to_device()) return -1;
    if (multi_ && !sync_label_table()) return -2; // sparse labels: no CSR table for the exact fold
    const size_t n = count_;
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_) dev_ctx_ = checkout();
    QueryCtx *c = dev_ctx_.get();
    if (!c) return -1;
    collect_dev_timing_locked();
    cudaStream_t st = s ? s : cudaStreamLegacy;
    const uint32_t nq32 = (uint32_t)nq, cap32 = (uint32_t)cap;
    const size_t qpitch = query_pitch();
    const CorpusView v = view();
    const int cmode = coarse_mode();
    const bool is8 = dtype_ == DT_I8 || dtype_ == DT_U8, is16 = dtype_ == DT_F16 || dtype_ == DT_BF16;
    // 1: the fp32 route of range_batch (same eligibility); 2: the fixed-radius pass over 8-bit rows, or the fixed-bound pass over
    // 16-bit rows with the margin eps16_q and CUDA-core rescoring (finite X only); 0: the exact scan only
    int path = 0;
    if (n > 0 && is8 && cmode != 0 && nq >= 16 && coarse_fixed_enabled() && coarse_supported(v, nq32, 1, CoarseDirect8) &&
        (!int_l2() || ensure_shadow(st))) {
        path = 2;
    } else if (n > 0 && is16 && cmode != 0 && nq >= 16 && coarse_fixed_enabled() && coarse_supported(v, nq32, 1, CoarseDirect16) &&
               ensure_shadow(st) && std::isfinite(shadow_max_norm_)) {
        path = 2;
    } else if (n > 0 && cmode == 1 && dtype_ == DT_F32 && !coarse_disabled_ && coarse_fixed_enabled() && coarse_supported(v, nq32, 1, CoarseF16) &&
               (nq >= 16 || single_query_takes_coarse(1)) && ensure_shadow(st) && shadow_values_in_range()) {
        path = 1;
    }
    const CoarseKind kind = path == 1 ? CoarseF16 : is16 ? CoarseDirect16 : CoarseDirect8;
    const CoarsePlan cp = path ? plan_coarse(v, nq32, kind, 1, 0, 1, 1) : CoarsePlan{};
    const WidePlan wp = n > 0 ? plan_topk_wide(v.n_rows, nq32) : WidePlan{};
    RangeScratch rs;
    uint32_t *d_ok, *d_idx, *d_n2, *d_total, *d_flags;
    const bool fold = multi_ && path; // a route's rows -> labels
    const auto layout = [&](void *base) {
        BatchScratch sc(base);
        if (path) rs.take(sc, *this, kind, cp, nq32, fold);
        d_total = sc.take<uint32_t>(1);
        d_ok = sc.take<uint32_t>(nq);  // reported flags
        d_idx = sc.take<uint32_t>(nq); // the open queries
        d_n2 = sc.take<uint32_t>(1);   // and their count
        d_flags = sc.take<uint32_t>(fold ? nq : 0); // multi-value: the reported flags (d_ok: 1 = folded, 0 = open)
        return sc.words();
    };
    if (!c->need_cand(layout(nullptr)) || (n > 0 && !c->need_scores(wp.score_elems))) return -1;
    layout(c->d_cand);
    LaunchCounters lc;
    uint64_t *comp = reinterpret_cast<uint64_t *>(d_labels);
    bool ok = cudaMemsetAsync(d_counts, 0, nq * 4, st) == cudaSuccess && cudaMemsetAsync(d_ok, 0, nq * 4, st) == cudaSuccess;
    // the timed span (VecSimB200_GetStats): the route's main pass, or the exact scan of a batch no route serves
    if (path)
        ok = ok && enqueue_range_route(*c, v, kind, cp, rs, d_q, qpitch, nq32, d_radii, nullptr, 0,
                                       RangeOut{comp, cap32, d_ok, d_counts, nullptr, d_total, fold ? d_flags : nullptr}, st, lc);
    if (n > 0) {
        // the exact scan: the queries a route left open (compacted on the device; none open = every launch exits at once), or all
        if (path) {
            ok = ok && launch_compact_unproven(d_ok, nq32, d_idx, d_n2, st) == cudaSuccess;
            lc.launches++;
        }
        if (!path) cudaEventRecord(c->ev_start, st);
        ok = ok && launch_range_wide(v, d_q, qpitch, nq32, path ? d_idx : nullptr, path ? d_n2 : nullptr, wp, c->d_scores, d_radii, cap32, comp,
                                     d_counts, c->d_abort, st, &lc, multi_ ? d_label_to_id_ : nullptr, multi_ ? d_label_rows_ : nullptr,
                                     multi_ ? (uint32_t)l2i_size_ : 0) == cudaSuccess;
        if (!path) cudaEventRecord(c->ev_stop, st);
    }
    ok = ok && launch_range_finish(d_labels, d_scores, d_counts, nq32, cap32, d_id_to_label_, order == BY_ID, st, &lc) == cudaSuccess;
    c->d_last_ok = fold ? d_flags : d_ok;
    c->last_ok_n = nq32;
    last_batch_coarse_ = true; // LastCoarseFlags: 1 = a tensor-core route answered the query, 0 = the exact scan, 3 = too many hit rows to fold
    last_batch_path_ = path;
    if (path) coarse_batches_++;
    dev_timing_pending_ = ok && n > 0;
    dev_timing_bytes_ = (uint64_t)n * stored_bytes_;
    launches_total_ += lc.launches;
    return ok ? 0 : -1;
}

double FlatIndex::distance_from(size_t label, const void *blob) {
    const double nan = std::numeric_limits<double>::quiet_NaN();
    std::vector<idType> ids;
    {
        std::lock_guard<std::mutex> g(mu_);
        if (multi_) {
            auto it = label_to_ids_.find(label);
            if (it == label_to_ids_.end()) return nan;
            ids = it->second;
        } else {
            auto it = label_to_id_.find(label);
            if (it == label_to_id_.end()) return nan;
            ids.push_back(it->second);
        }
    }
    if (!flush()) return nan;
    auto c = checkout();
    if (!c) return nan;
    LaunchCounters lc;
    bool ok = c->need_ids(ids.size()) && stage_queries(*c, blob, 0, 1, false);
    if (ok) {
        for (size_t i = 0; i < ids.size(); i++) c->h_ids[i] = ids[i];
        ok = cudaMemcpyAsync(c->d_ids, c->h_ids, ids.size() * 4, cudaMemcpyHostToDevice, c->stream) == cudaSuccess;
    }
    ok = ok && launch_gather_distances(view(), c->d_query, c->d_ids, (uint32_t)ids.size(), c->d_dist, c->stream, &lc) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(c->h_dist, c->d_dist, ids.size() * 4, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c->stream) == cudaSuccess;
    double best = nan;
    if (ok) { // brute_force_multi.h:224-241, the same fold as gather_min_kernel: a NaN row survives only in the last place
        float dist = std::numeric_limits<float>::infinity();
        for (size_t i = 0; i < ids.size(); i++) dist = (dist < c->h_dist[i]) ? dist : c->h_dist[i];
        best = (double)dist;
    }
    launches_total_ += lc.launches;
    checkin(std::move(c));
    return best;
}

// brute_force.h:380-451, thresholds and float/double comparison types reproduced exactly.
bool FlatIndex::prefer_adhoc(size_t subset, size_t k, bool initial) {
    (void)k;
    const size_t index_size = count_;
    subset = std::min(subset, index_size);
    const size_t d = dim_;
    const float r = (index_size == 0) ? 0.0f : (float)subset / (float)label_count();
    bool res;
    if (index_size <= 5500) {
        res = true;
    } else if (d <= 300) {
        if (r <= 0.15)
            res = true;
        else if (r <= 0.35)
            res = (d <= 75) ? false : (index_size <= 550000);
        else
            res = false;
    } else {
        if (r <= 0.55)
            res = true;
        else if (d <= 750)
            res = false;
        else
            res = (r <= 0.75);
    }
    last_mode_ = res ? (initial ? HYBRID_ADHOC_BF : HYBRID_BATCHES_TO_ADHOC_BF) : HYBRID_BATCHES;
    return res;
}

// ------------------------------------------------------------------------------------------------
// batch iterator
// ------------------------------------------------------------------------------------------------
BatchIter *FlatIndex::batch_new(const void *q, VecSimQueryParams *qp) {
    auto *it = new BatchIter();
    it->index = this;
    it->query.assign(query_pitch(), 0);
    preprocess_query(q, it->query.data()); // forced copy, brute_force.h:371-372
    it->timeout_ctx = qp ? qp->timeoutCtx : nullptr;
    it->label_count = label_count();
    return it;
}

VecSimQueryReply *FlatIndex::batch_next(BatchIter *it, size_t n_res, VecSimQueryReply_Order order) {
    auto *rep = new VecSimQueryReply();
    if (!it->scored) {
        // first call: the only time the index is read (bf_batch_iterator.h:176-189)
        if (!flush()) return rep;
        it->n_rows = (uint32_t)count_;
        it->label_count = label_count();
        it->id_to_label_snap = id_to_label_;
        if (timed_out(it->timeout_ctx)) {
            rep->code = VecSim_QueryReply_TimedOut;
            return rep;
        }
        if (!it->ctx) it->ctx = checkout();
        if (!it->ctx) return rep;
        if (it->n_rows) {
            LaunchCounters lc;
            bool ok = it->ctx->need_scores(it->n_rows) && stage_queries(*it->ctx, it->query.data(), 0, 1, false);
            ok = ok && launch_scan_scores(view(), it->ctx->d_query, it->ctx->d_scores, it->ctx->stream, &lc) == cudaSuccess;
            ok = ok && cudaStreamSynchronize(it->ctx->stream) == cudaSuccess;
            launches_total_ += lc.launches;
            record_scan(nullptr, (uint64_t)it->n_rows * stored_bytes_);
            if (!ok) return rep;
        }
        it->scored = true;
    }
    if (timed_out(it->timeout_ctx)) {
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    const size_t remaining_labels = it->label_count - it->returned;
    const size_t want_labels = std::min(n_res, remaining_labels);
    size_t produced = 0;
    while (produced < want_labels) {
        const size_t want = multi_ ? std::max<size_t>(2 * (want_labels - produced), 64) : (want_labels - produced);
        const long got = select_from_scores(*it->ctx, it->n_rows, it->has_cursor, it->cursor, std::min<size_t>(want, it->n_rows));
        if (got <= 0) break;
        for (long i = 0; i < got; i++) {
            const uint64_t comp = it->ctx->h_out[i];
            if (produced < want_labels) {
                const VecSimQueryResult r = decode(comp, it->id_to_label_snap);
                it->has_cursor = true;
                it->cursor = comp;
                if (multi_ && !it->seen.insert(r.id).second) continue;
                rep->results.push_back(r);
                produced++;
            } else {
                break; // leave the rest for the next call: cursor stays on the last consumed entry
            }
        }
        if ((size_t)got < std::min<size_t>(want, it->n_rows)) break;
    }
    it->returned += rep->results.size();
    finish_reply(rep, order == BY_ID ? BY_ID : BY_SCORE);
    return rep;
}

// ------------------------------------------------------------------------------------------------
// ad-hoc context
// ------------------------------------------------------------------------------------------------
AdhocCtx *FlatIndex::adhoc_new(const void *q) {
    auto *a = new AdhocCtx();
    a->index = this;
    a->query.assign(stored_bytes_, 0);
    preprocess_query(q, a->query.data()); // the context normalises internally (hybrid_reader.c:212-214)
    a->ctx = checkout();
    if (!a->ctx) {
        delete a;
        return nullptr;
    }
    return a;
}

void FlatIndex::adhoc_distances(AdhocCtx *a, const size_t *labels, double *out, size_t n) {
    const double nan = std::numeric_limits<double>::quiet_NaN();
    for (size_t i = 0; i < n; i++) out[i] = nan;
    if (n == 0 || !flush()) return;
    QueryCtx &c = *a->ctx;
    LaunchCounters lc;
    // expand labels to row ids (multi: several rows per label, folded on the host as getDistanceFrom_Unsafe folds them)
    std::vector<uint32_t> ids;
    std::vector<uint32_t> owner;
    ids.reserve(n);
    {
        std::lock_guard<std::mutex> g(mu_);
        for (size_t i = 0; i < n; i++) {
            if (multi_) {
                auto it = label_to_ids_.find(labels[i]);
                if (it == label_to_ids_.end()) continue;
                for (idType id : it->second) {
                    ids.push_back(id);
                    owner.push_back((uint32_t)i);
                }
            } else {
                auto it = label_to_id_.find(labels[i]);
                if (it == label_to_id_.end()) continue;
                ids.push_back(it->second);
                owner.push_back((uint32_t)i);
            }
        }
    }
    if (ids.empty()) return;
    bool ok = c.need_ids(ids.size());
    if (ok && !a->query_on_device) {
        ok = stage_queries(c, a->query.data(), 0, 1, false);
        a->query_on_device = ok;
    }
    if (ok) {
        memcpy(c.h_ids, ids.data(), ids.size() * 4);
        ok = cudaMemcpyAsync(c.d_ids, c.h_ids, ids.size() * 4, cudaMemcpyHostToDevice, c.stream) == cudaSuccess;
    }
    ok = ok && launch_gather_distances(view(), c.d_query, c.d_ids, (uint32_t)ids.size(), c.d_dist, c.stream, &lc) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(c.h_dist, c.d_dist, ids.size() * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c.stream) == cudaSuccess;
    launches_total_ += lc.launches;
    if (!ok) return;
    // brute_force_multi.h:234-238 per label, over its rows in order: dist = +inf, then dist = (dist < d) ? dist : d.  A NaN row
    // resets dist to NaN and the next row replaces it, so only a NaN in the last row survives (gather_min_kernel's fold)
    std::vector<float> fold(n, std::numeric_limits<float>::infinity());
    for (size_t i = 0; i < ids.size(); i++) {
        float &f = fold[owner[i]];
        f = (f < c.h_dist[i]) ? f : c.h_dist[i];
    }
    for (size_t i = 0; i < ids.size(); i++) out[owner[i]] = (double)fold[owner[i]];
}


// ------------------------------------------------------------------------------------------------
// fused hybrid ad-hoc query (HybridIterator in HYBRID_ADHOC_BF mode, src/iterators/hybrid_reader.c:289-335:
// child docIds in ascending order -> GetDistanceFrom each -> heap of the k best, strict `<` admission, NaN = deleted)
// ------------------------------------------------------------------------------------------------
bool FlatIndex::sync_label_table() {
    std::lock_guard<std::mutex> g(mu_);
    if (!l2i_dirty_ && d_label_to_id_) return true;
    size_t max_label = 0;
    for (size_t i = 0; i < count_; i++) max_label = std::max(max_label, id_to_label_[i]);
    if (max_label > 4 * count_ + (1u << 24) || max_label >= 0xFFFFFFFFull) return false; // sparse labels: no dense table
    const size_t size = max_label + 1;
    // single-value: row of each label (0xFFFFFFFF = absent); multi-value: CSR offsets [size + 1] over `rows`
    const size_t entries = multi_ ? size + 1 : size;
    std::vector<uint32_t> tab(entries, multi_ ? 0u : 0xFFFFFFFFu);
    std::vector<uint32_t> rows;
    if (multi_) {
        for (const auto &kv : label_to_ids_) tab[kv.first + 1] = (uint32_t)kv.second.size();
        for (size_t l = 0; l < size; l++) tab[l + 1] += tab[l];
        rows.resize(count_);
        for (const auto &kv : label_to_ids_)
            std::copy(kv.second.begin(), kv.second.end(), rows.begin() + tab[kv.first]);
    } else {
        for (size_t i = 0; i < count_; i++) tab[id_to_label_[i]] = (uint32_t)i;
    }
    if (entries > l2i_cap_) {
        cudaFree(d_label_to_id_);
        d_label_to_id_ = nullptr;
        const size_t cap = entries + entries / 4 + 1024;
        CU_OK(cudaMalloc(&d_label_to_id_, cap * 4));
        l2i_cap_ = cap;
    }
    CU_OK(cudaMemcpy(d_label_to_id_, tab.data(), entries * 4, cudaMemcpyHostToDevice));
    if (multi_) {
        if (rows.size() > label_rows_cap_ || !d_label_rows_) {
            cudaFree(d_label_rows_);
            d_label_rows_ = nullptr;
            const size_t cap = rows.size() + rows.size() / 4 + 1024;
            CU_OK(cudaMalloc(&d_label_rows_, cap * 4));
            label_rows_cap_ = cap;
        }
        CU_OK(cudaMemcpy(d_label_rows_, rows.data(), rows.size() * 4, cudaMemcpyHostToDevice));
    }
    l2i_size_ = size;
    l2i_dirty_ = false;
    return true;
}

int FlatIndex::topk_filtered(const void *q, size_t k, const uint32_t *doc_ids, size_t n, bool ids_on_device, size_t *out_labels,
                             double *out_scores, size_t *out_count) {
    *out_count = 0;
    last_mode_ = HYBRID_ADHOC_BF;
    if (k == 0 || n == 0) return 0;
    if (n > 0xFFFFFFF0ull) return -2;
    if (!flush()) return -1;
    if (count_ == 0) return 0;
    if (!sync_label_table()) return -2;
    auto c = checkout();
    if (!c) return -1;
    LaunchCounters lc;
    bool ok = c->need_ids(2 * n + 256) && c->need_scores(n) && stage_queries(*c, q, 0, 1, true);
    // d_ids: [0,n) row ids, [n,2n) the labels when they arrive from the host
    const uint32_t *d_labels = doc_ids;
    if (ok && !ids_on_device) {
        ok = cudaMemcpyAsync(c->d_ids + n, doc_ids, n * 4, cudaMemcpyHostToDevice, c->stream) == cudaSuccess;
        d_labels = c->d_ids + n;
    }
    if (multi_) { // one score per docId: the min fold over its rows (DESIGN.md §4.4)
        ok = ok && launch_gather_min_distances(view(), c->d_query, d_labels, (uint32_t)n, d_label_to_id_, (uint32_t)l2i_size_, d_label_rows_,
                                               c->d_scores, c->stream, &lc) == cudaSuccess;
    } else {
        ok = ok && launch_map_labels(d_labels, (uint32_t)n, d_label_to_id_, (uint32_t)l2i_size_, c->d_ids, c->stream, &lc) == cudaSuccess;
        ok = ok && launch_gather_distances(view(), c->d_query, c->d_ids, (uint32_t)n, c->d_scores, c->stream, &lc) == cudaSuccess;
    }
    launches_total_ += lc.launches;
    if (!ok) {
        checkin(std::move(c));
        return -1;
    }
    // k best positions by (distance asc, position asc) = (distance, docId): NaN (deleted docs) sort last and are dropped
    const size_t want = std::min(k, n);
    const long got = select_from_scores(*c, (uint32_t)n, false, 0, want);
    if (got < 0) {
        checkin(std::move(c));
        return -1;
    }
    LaunchCounters lc2;
    uint32_t *d_sel = c->d_ids; // row ids are no longer needed
    ok = launch_pick_labels(c->d_out, (uint32_t)got, d_labels, d_sel, c->stream, &lc2) == cudaSuccess;
    ok = ok && cudaMemcpyAsync(c->h_ids, d_sel, (size_t)got * 4, cudaMemcpyDeviceToHost, c->stream) == cudaSuccess;
    ok = ok && cudaStreamSynchronize(c->stream) == cudaSuccess;
    launches_total_ += lc2.launches;
    size_t w = 0;
    if (ok)
        for (long i = 0; i < got; i++) {
            const float d = key_to_float((uint32_t)(c->h_out[i] >> 32));
            if (std::isnan(d)) continue;
            out_labels[w] = c->h_ids[i];
            out_scores[w] = (double)d;
            w++;
        }
    *out_count = w;
    checkin(std::move(c));
    return ok ? 0 : -1;
}


// The same for MANY queries (BASELINE configs[4]: a batch of hybrid queries, each with its own filter set): every query's chain
// (labels -> rows, gathered distances, selection, label pick, D2H) is enqueued on its own context's stream before anything is
// waited for, so the chains overlap and the host pays one round of synchronisations instead of two per query.  Device-resident
// id lists only (the filters' AND / OR results).
int FlatIndex::topk_filtered_batch(const void *const *queries, size_t nq, size_t k, const uint32_t *const *d_doc_ids, const size_t *counts,
                                   size_t *out_labels, double *out_scores, size_t *out_counts) {
    for (size_t i = 0; i < nq; i++) out_counts[i] = 0;
    last_mode_ = HYBRID_ADHOC_BF;
    if (k == 0 || nq == 0) return 0;
    if (k > (size_t)kMaxFusedK) return -2;
    if (!flush()) return -1;
    if (count_ == 0) return 0;
    if (!sync_label_table()) return -2;
    constexpr size_t kWave = 16; // contexts in flight at once
    int rc = 0;
    for (size_t q0 = 0; q0 < nq && rc == 0; q0 += kWave) {
        const size_t q1 = std::min(nq, q0 + kWave);
        struct Job {
            std::unique_ptr<QueryCtx> c;
            size_t want = 0;
            bool ok = false;
        };
        std::vector<Job> jobs(q1 - q0);
        LaunchCounters lc;
        for (size_t qi = q0; qi < q1; qi++) {
            Job &j = jobs[qi - q0];
            const size_t n = counts[qi];
            if (n == 0) continue;
            if (n > 0xFFFFFFF0ull) {
                rc = -2;
                break;
            }
            j.c = checkout();
            if (!j.c) {
                rc = -1;
                break;
            }
            QueryCtx &c = *j.c;
            j.want = std::min(k, n);
            const uint32_t lists = plan_select_scores_lists((uint32_t)n);
            bool ok = c.need_ids(2 * n + 256) && c.need_scores(n) && c.need_out(j.want + 1) && c.need_cand((size_t)lists * j.want) &&
                      stage_queries(c, queries[qi], 0, 1, true);
            const uint32_t *d_labels = d_doc_ids[qi];
            if (multi_) {
                ok = ok && launch_gather_min_distances(view(), c.d_query, d_labels, (uint32_t)n, d_label_to_id_, (uint32_t)l2i_size_,
                                                       d_label_rows_, c.d_scores, c.stream, &lc) == cudaSuccess;
            } else {
                ok = ok && launch_map_labels(d_labels, (uint32_t)n, d_label_to_id_, (uint32_t)l2i_size_, c.d_ids, c.stream, &lc) == cudaSuccess;
                ok = ok && launch_gather_distances(view(), c.d_query, c.d_ids, (uint32_t)n, c.d_scores, c.stream, &lc) == cudaSuccess;
            }
            ok = ok && launch_select_scores(c.d_scores, (uint32_t)n, nullptr, (uint32_t)j.want, c.d_cand, c.stream, &lc) == cudaSuccess;
            ok = ok && launch_final_select(c.d_cand, 1, lists * (uint32_t)j.want, (uint32_t)j.want, c.d_out, c.stream, &lc) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(c.h_out, c.d_out, j.want * 8, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
            // the selected positions -> labels (empty slots pick nothing that is read back: they are cut below)
            ok = ok && launch_pick_labels(c.d_out, (uint32_t)j.want, d_labels, c.d_ids, c.stream, &lc) == cudaSuccess;
            ok = ok && cudaMemcpyAsync(c.h_ids, c.d_ids, j.want * 4, cudaMemcpyDeviceToHost, c.stream) == cudaSuccess;
            j.ok = ok;
            if (!ok) rc = -1;
        }
        launches_total_ += lc.launches;
        for (size_t qi = q0; qi < q1; qi++) { // one round of waits; contexts go back even on failure
            Job &j = jobs[qi - q0];
            if (!j.c) continue;
            const bool synced = cudaStreamSynchronize(j.c->stream) == cudaSuccess;
            if (j.ok && synced && rc == 0) {
                size_t w = 0;
                for (size_t i = 0; i < j.want; i++) {
                    if (j.c->h_out[i] == kEmptySlot) break;
                    const float d = key_to_float((uint32_t)(j.c->h_out[i] >> 32));
                    if (std::isnan(d)) continue;
                    out_labels[qi * k + w] = j.c->h_ids[i];
                    out_scores[qi * k + w] = (double)d;
                    w++;
                }
                out_counts[qi] = w;
            } else if (!synced) {
                rc = -1;
            }
            checkin(std::move(j.c));
        }
    }
    return rc;
}

// dev_mu_ held: a staging slot of at least `elems` words whose previous upload has executed (a never-recorded event counts as
// complete), else a new one; NULL on an allocation failure
FlatIndex::TableSlot *FlatIndex::table_slot(size_t elems) {
    for (TableSlot &t : table_ring_)
        if (t.cap >= elems && cudaEventQuery(t.ev) == cudaSuccess) {
            cudaGetLastError();
            return &t;
        }
    cudaGetLastError(); // cudaErrorNotReady of a slot in flight is no failure
    TableSlot t;
    t.cap = std::max<size_t>(2 * elems, 1024);
    if (cudaMallocHost(&t.h, t.cap * 8) != cudaSuccess) return nullptr;
    if (cudaEventCreateWithFlags(&t.ev, cudaEventDisableTiming) != cudaSuccess) {
        cudaFreeHost(t.h);
        return nullptr;
    }
    table_ring_.push_back(t);
    return &table_ring_.back();
}

// The caps of a ragged batch: their sum, their largest and the gather's chunks.  ok = false when a cap exceeds 0xFFFFFFF0 (the entry
// points return -2)
struct RaggedCaps {
    bool ok = true;
    size_t total = 0, max_cap = 0;
    uint64_t blocks = 0;
};
static RaggedCaps scan_caps(const size_t *caps, size_t nq) {
    RaggedCaps r;
    for (size_t i = 0; i < nq; i++) {
        if (caps[i] > 0xFFFFFFF0ull) {
            r.ok = false;
            return r;
        }
        r.total += caps[i];
        r.max_cap = std::max(r.max_cap, caps[i]);
        r.blocks += ragged_blocks(caps[i]);
    }
    return r;
}

bool FlatIndex::upload_ragged_table(uint64_t *d_tab, const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                    uint32_t nq, const std::vector<uint32_t> &tail, cudaStream_t st, RaggedBatch &b, bool &ok) {
    const size_t elems = ragged_table_elems(nq, tail.size());
    TableSlot *slot = table_slot(elems);
    if (!slot) return false;
    uint64_t *h = slot->h, off = 0, blk = 0;
    for (size_t i = 0; i < nq; i++) {
        h[i] = (uint64_t)(uintptr_t)d_doc_ids[i];
        h[nq + i] = d_counts ? (uint64_t)(uintptr_t)d_counts[i] : 0;
        h[2 * nq + i] = off;
        h[3 * nq + 1 + i] = blk;
        off += caps[i];
        blk += ragged_blocks(caps[i]);
    }
    h[3 * nq] = off;
    h[4 * nq + 1] = blk;
    if (!tail.empty()) memcpy(h + 4 * nq + 2, tail.data(), tail.size() * sizeof(uint32_t));
    ok = ok && cudaMemcpyAsync(d_tab, h, elems * 8, cudaMemcpyHostToDevice, st) == cudaSuccess;
    ok = ok && cudaEventRecord(slot->ev, st) == cudaSuccess;
    b = RaggedBatch{reinterpret_cast<const uint32_t *const *>(d_tab), reinterpret_cast<const uint32_t *const *>(d_tab + nq), d_tab + 2 * nq, nq};
    return true;
}

// The same batch with device pointers end to end (DESIGN.md §4.6): no filter length comes back to the host.  One ragged gather over
// the flat space of the caps, 2 ceil(k / 128) segmented selects, one unpack: 2 + 2 ceil(k / 128) launches whatever nq.  Selection is
// by (distance, position in the filter) as in topk_filtered, so every row equals its answer.
int FlatIndex::topk_filtered_batch_device(const void *d_q, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                          const uint32_t *const *d_counts, const size_t *caps, int64_t *d_labels, float *d_scores,
                                          uint32_t *d_counts_out, cudaStream_t s) {
    last_mode_ = HYBRID_ADHOC_BF;
    if (nq == 0 || k == 0) return 0;
    if (k > (size_t)kMaxWideK || nq > 0x7FFFFFFFull) return -1;
    const RaggedCaps rc = scan_caps(caps, nq);
    if (!rc.ok) return -2;
    if (!flush()) return -1;
    if (!sync_label_table()) return -2;
    const uint32_t nq32 = (uint32_t)nq, chunk = (uint32_t)std::min<size_t>(k, kMaxFusedK);
    const uint32_t parts = plan_ragged_select_parts(rc.max_cap, nq32);
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_) dev_ctx_ = checkout();
    QueryCtx *c = dev_ctx_.get();
    if (!c) return -1;
    const size_t tab_elems = ragged_table_elems(nq, 0);
    uint64_t *tab, *cand, *out;
    float *scores;
    const auto layout = [&](void *base) {
        BatchScratch sc(base);
        tab = sc.take<uint64_t>(tab_elems);
        scores = sc.take<float>(rc.total);
        cand = sc.take<uint64_t>((size_t)nq * parts * 8 * chunk); // 8 lists (one per warp) per select CTA
        out = sc.take<uint64_t>(nq * k);
        return sc.words();
    };
    if (!c->need_cand(layout(nullptr))) return -1;
    layout(c->d_cand);
    cudaStream_t st = s ? s : cudaStreamLegacy; // NULL = the legacy default stream, as everywhere in CUDA
    RaggedBatch b;
    bool ok = true;
    if (!upload_ragged_table(tab, d_doc_ids, d_counts, caps, nq32, {}, st, b, ok)) return -1;
    LaunchCounters lc;
    ok = ok && launch_gather_ragged(view(), d_q, query_pitch(), b, tab + 3 * nq + 1, rc.blocks, d_label_to_id_, (uint32_t)l2i_size_,
                                    multi_ ? d_label_rows_ : nullptr, scores, st, &lc) == cudaSuccess;
    ok = ok && launch_topk_ragged(b, scores, (uint32_t)k, parts, cand, out, st, &lc) == cudaSuccess;
    ok = ok && launch_unpack_ragged(b, out, (uint32_t)k, d_labels, d_scores, d_counts_out, st, &lc) == cudaSuccess;
    launches_total_ += lc.launches;
    return ok ? 0 : -1;
}

// Mode choice of a hybrid batch (DESIGN.md §4.10), from what the host already knows.  A query can take the dense route when its cap
// lets the sample pass meet enough filtered rows: at a filtered fraction f = cap / n the sample must visit tiles_per_k * k / f row
// tiles, and that must stay within a quarter of the corpus, so cap >= 4 * tiles_per_k * k * 128 (rows per tile).  Those queries
// take it together when the bytes their gathers would read exceed what the dense route reads: the shadow once (+ the sample
// pass), the bitmaps and their lists.
static constexpr double kHybridSampleShare = 0.25;
static double hybrid_tiles_per_k(uint32_t ke) { return ke > kCoarseMaxK ? 1 / 32.0 : 2.0; }
static size_t hybrid_cap_floor(uint32_t ke) { return (size_t)std::ceil(hybrid_tiles_per_k(ke) * ke * 128 / kHybridSampleShare); }

int FlatIndex::hybrid_topk_batch_device(const void *d_q, size_t nq, size_t k, const uint32_t *const *d_doc_ids,
                                        const uint32_t *const *d_counts, const size_t *caps, VecSimQueryParams *qp, int64_t *d_labels,
                                        float *d_scores, uint32_t *d_counts_out, int *out_modes, cudaStream_t s) {
    const int policy = qp ? (int)qp->searchMode : (int)EMPTY_MODE;
    if (policy != EMPTY_MODE && policy != HYBRID_ADHOC_BF && policy != HYBRID_BATCHES) return -1;
    if (out_modes)
        for (size_t i = 0; i < nq; i++) out_modes[i] = HYBRID_ADHOC_BF;
    last_mode_ = HYBRID_ADHOC_BF;
    if (nq == 0 || k == 0) return 0;
    if (k > (size_t)kMaxWideK || nq > 0x7FFFFFFFull) return -1;
    const RaggedCaps rc = scan_caps(caps, nq);
    if (!rc.ok) return -2;
    if (!flush()) return -1;
    if (!sync_label_table()) return -2;
    const size_t n = count_;
    const uint32_t nq32 = (uint32_t)nq, ke = (uint32_t)std::min<size_t>(k, std::max<size_t>(n, 1));
    cudaStream_t st = s ? s : cudaStreamLegacy; // NULL = the legacy default stream, as everywhere in CUDA
    const CorpusView v = view();
    const bool unit = unit_rows();
    // the dense route: the fp32 two-pass route of §4.5 over the fp16 shadow (L2 / raw inner product: its norm-scaled bound)
    const bool eligible = policy != HYBRID_ADHOC_BF && !multi_ && dtype_ == DT_F32 && coarse_mode() == 1 && coarse_fixed_enabled() &&
                          !coarse_disabled_ && n >= 65536 && coarse_supported(v, 16, ke, CoarseF16);
    std::vector<uint32_t> dense_q;
    if (eligible) {
        const size_t floor_cap = policy == HYBRID_BATCHES ? 0 : hybrid_cap_floor(ke);
        double gather_bytes = 0, list_bytes = 0;
        for (size_t i = 0; i < nq; i++)
            if (caps[i] >= floor_cap) {
                dense_q.push_back((uint32_t)i);
                gather_bytes += (double)caps[i] * (double)(stored_bytes_ + 8);
                list_bytes += (double)caps[i] * 8;
            }
        if (policy != HYBRID_BATCHES && !dense_q.empty()) {
            const double shadow = (double)n * dim_ * 2 * (1 + kHybridSampleShare), bitmaps = (double)dense_q.size() * ((n + 31) / 32) * 4 * 2;
            if (!(gather_bytes > shadow + bitmaps + list_bytes)) dense_q.clear();
        }
        // a subset below the batch route's own 16 queries does not pay for a first shadow build
        if (dense_q.size() < 16 && !d_shadow_) dense_q.clear();
        if (!dense_q.empty() && !ensure_shadow(st)) dense_q.clear();
        if (!dense_q.empty() && !shadow_values_in_range()) dense_q.clear();
        if (!dense_q.empty() && !sync_labels_to_device()) return -1;
    }
    const uint32_t nd = (uint32_t)dense_q.size();
    if (out_modes)
        for (uint32_t p : dense_q) out_modes[p] = HYBRID_BATCHES;
    last_mode_ = nd ? HYBRID_BATCHES : HYBRID_ADHOC_BF;
    const uint32_t chunk = (uint32_t)std::min<size_t>(k, kMaxFusedK);
    const uint32_t parts = plan_ragged_select_parts(rc.max_cap, nq32);
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_) dev_ctx_ = checkout();
    QueryCtx *c = dev_ctx_.get();
    if (!c) return -1;
    // dense-route plans (positions 0 .. nd - 1 = the dense queries in batch order)
    KnnTiers t;
    const uint32_t words = (uint32_t)((n + 31) / 32);
    if (nd) {
        // the sample must hold a few times k FILTERED rows: at the smallest filtered fraction among the dense queries it visits
        // tiles_per_k / f times the tiles of the unfiltered route (caps bound the counts from above: a low count only costs time)
        double fmin = 1.0;
        for (uint32_t q : dense_q) fmin = std::min(fmin, std::max((double)caps[q] / (double)n, 1e-9));
        t = plan_knn_tiers(v, nd, CoarseF16, ke, ke > kCoarseMaxK ? 128.0 : 24.0, hybrid_tiles_per_k(ke) / fmin, true);
    }
    const size_t qpitch = query_pitch();
    // u32 words after the pinned table: [dense queries nd][dense count 1][dense position of each query nq]
    std::vector<uint32_t> tail(dense_q);
    tail.push_back(nd);
    tail.resize(nd + 1 + nq, 0xFFFFFFFFu);
    for (uint32_t p = 0; p < nd; p++) tail[nd + 1 + dense_q[p]] = p;
    const size_t tab_elems = ragged_table_elems(nq, tail.size());
    uint64_t *tab, *cand, *out, *out_d;
    float *scores;
    uint8_t *q32;
    uint32_t *bm, *d_flags, *d_live;
    const uint32_t **d_live_ptr;
    KnnScratch ks;
    const auto layout = [&](void *base) {
        BatchScratch sc(base);
        tab = sc.take<uint64_t>(tab_elems);
        scores = sc.take<float>(rc.total);
        cand = sc.take<uint64_t>((size_t)nq * parts * 8 * chunk); // 8 lists (one per warp) per select CTA
        out = sc.take<uint64_t>(nq * k);
        d_flags = sc.take<uint32_t>(nq);
        d_live = sc.take<uint32_t>(nd ? nq : 0);
        d_live_ptr = sc.take<const uint32_t *>(nd ? nq : 0);
        bm = sc.take<uint32_t>((size_t)nd * words);
        q32 = sc.take<uint8_t>((size_t)nd * qpitch);
        ks.take(sc, t, nd, f16_query_pitch(), !unit, false);
        out_d = sc.take<uint64_t>((size_t)nd * ke);
        return sc.words();
    };
    if (!c->need_cand(layout(nullptr))) return -1;
    layout(c->d_cand);
    RaggedBatch b;
    bool ok = true;
    if (!upload_ragged_table(tab, d_doc_ids, d_counts, caps, nq32, tail, st, b, ok)) return -1;
    const uint32_t *d_dense_q = reinterpret_cast<const uint32_t *>(tab + 4 * nq + 2), *d_nd = d_dense_q + nd, *d_pos = d_nd + 1;
    LaunchCounters lc;
    DenseRows dr;
    RaggedBatch bg = b; // the gather's batch: every query, or (dense route) the open ones
    if (nd) {
        // 1. row-space filter bitmaps of the dense queries; their queries packed to the front (fp32 for the rescoring, fp16 for the GEMM)
        ok = ok && cudaMemsetAsync(bm, 0, (size_t)nd * words * 4, st) == cudaSuccess;
        ok = ok && launch_filter_bitmaps(b, d_dense_q, nd, rc.max_cap, d_label_to_id_, (uint32_t)l2i_size_, bm, words, st, &lc) == cudaSuccess;
        ok = ok && launch_gather_queries(d_q, qpitch, nullptr, d_dense_q, d_nd, nd, q32, nullptr, st) == cudaSuccess;
        lc.launches++;
        CoarseOperands ops{};
        ok = ok && shadow_operands(q32, qpitch, nd, ks.q, ks.qn2, st, lc, ops);
        // 2. sample pass over the filtered rows and the bound; 3. main pass; 4. exact rescoring + proof, selected by (distance, docId);
        // 5. second tier for the queries whose lists overflowed: adaptive lists of 128 over the filtered rows
        ok = ok && enqueue_knn_tiers(*c, v, CoarseF16, t, ks, ops, q32, qpitch, nd, ke, out_d, bm, words, d_id_to_label_, st, lc);
        // 6. the gather answers the ad-hoc queries and the dense ones still open; a proven query's count is 0
        ok = ok && launch_hybrid_open(b, d_pos, ks.ok, d_flags, d_live, d_live_ptr, st, &lc) == cudaSuccess;
        bg.counts = d_live_ptr;
        dr = DenseRows{out_d, d_pos, d_flags};
    } else {
        ok = ok && cudaMemsetAsync(d_flags, 0, nq * 4, st) == cudaSuccess;
    }
    // with dense queries in the batch most chunks of the caps are empty: a grid of a few CTAs per SM strides over them
    const uint64_t max_grid = nd ? (uint64_t)device_sm_count() * 16 : 0;
    ok = ok && launch_gather_ragged(v, d_q, qpitch, bg, tab + 3 * nq + 1, rc.blocks, d_label_to_id_, (uint32_t)l2i_size_,
                                    multi_ ? d_label_rows_ : nullptr, scores, st, &lc, max_grid) == cudaSuccess;
    ok = ok && launch_topk_ragged(bg, scores, (uint32_t)k, parts, cand, out, st, &lc) == cudaSuccess;
    // 7. one unpack: gather rows map positions to docIds, proven dense rows carry them
    ok = ok && launch_unpack_ragged(b, out, (uint32_t)k, d_labels, d_scores, d_counts_out, st, &lc, dr) == cudaSuccess;
    c->d_last_ok = d_flags;
    c->last_ok_n = nq32;
    last_batch_coarse_ = true;
    last_batch_path_ = nd ? 1 : 0;
    if (nd) coarse_batches_++;
    launches_total_ += lc.launches;
    return ok ? 0 : -1;
}

// Mode choice of a filtered range batch (DESIGN.md §4.13), from what the host already knows.  There is no sample pass, so no cap
// floor: the batch takes a dense route as a whole when the bytes its gathers would read exceed what the dense route reads, the
// rows of its main pass (`pass_bytes`), two passes over one row bitmap per query, and the lists.
static constexpr size_t kHybridRangeMinDense = 16; // queries below which a dense route does not pay for its first shadow / table
static bool hybrid_range_dense_pays(size_t cap_sum, size_t stored_bytes, double pass_bytes, size_t nq, size_t n) {
    const double gather = (double)cap_sum * (double)(stored_bytes + 8), bitmaps = (double)nq * ((n + 31) / 32) * 4 * 2;
    return gather > pass_bytes + bitmaps + 8.0 * (double)cap_sum;
}

// Filtered range batches (DESIGN.md §4.13): range_device's answer for each query restricted to its filter.  Either every query takes
// the range form of the ragged gather, or the whole batch takes one of range_device's routes with the filter bitmaps applied to the
// rows of its main pass; the gather then answers the queries that route left open.  Hits are gathered as (score key, row)
// composites in d_labels itself and ordered by range_finish, as in range_device.  Launches: 2 on the gather alone; the fp32 route
// 8 (+1 for L2 / inner product), the 8-bit route 6 (+1 for L2).
int FlatIndex::hybrid_range_batch_device(const void *d_q, size_t nq, const float *d_radii, size_t cap, VecSimQueryReply_Order order,
                                         const uint32_t *const *d_doc_ids, const uint32_t *const *d_counts, const size_t *caps,
                                         VecSimQueryParams *qp, int64_t *d_labels, float *d_scores, uint32_t *d_counts_out, int *out_modes,
                                         cudaStream_t s) {
    const int policy = qp ? (int)qp->searchMode : (int)EMPTY_MODE;
    if (policy != EMPTY_MODE && policy != HYBRID_ADHOC_BF && policy != HYBRID_BATCHES) return -1;
    if (cap == 0 || cap > kRangeDeviceMaxCap || (order != BY_ID && order != BY_SCORE) || nq > 0x7FFFFFFFull) return -1;
    if (out_modes)
        for (size_t i = 0; i < nq; i++) out_modes[i] = HYBRID_ADHOC_BF;
    last_mode_ = RANGE_QUERY;
    if (nq == 0) return 0;
    const RaggedCaps rc = scan_caps(caps, nq);
    if (!rc.ok) return -2;
    if (!flush()) return -1;
    if (!sync_label_table()) return -2;
    if (!sync_labels_to_device()) return -1;
    const size_t n = count_;
    const uint32_t nq32 = (uint32_t)nq, cap32 = (uint32_t)cap;
    cudaStream_t st = s ? s : cudaStreamLegacy; // NULL = the legacy default stream, as everywhere in CUDA
    const CorpusView v = view();
    const int cmode = coarse_mode();
    // 1: range_device's fp32 route, 2: its 8-bit fixed-radius route (each with range_device's eligibility), 0: the gather only
    int path = 0;
    if (policy != HYBRID_ADHOC_BF && !multi_ && n > 0 && coarse_fixed_enabled()) {
        const bool r8 = (dtype_ == DT_I8 || dtype_ == DT_U8) && cmode != 0 && nq >= kHybridRangeMinDense &&
                        coarse_supported(v, nq32, 1, CoarseDirect8);
        const bool r32 = dtype_ == DT_F32 && cmode == 1 && !coarse_disabled_ && coarse_supported(v, nq32, 1, CoarseF16) &&
                         (nq >= kHybridRangeMinDense || single_query_takes_coarse(1));
        const double pass_bytes = (double)n * dim_ * (r8 ? 1 : 2); // the 8-bit rows, or the fp16 shadow
        if ((r8 || r32) && (policy == HYBRID_BATCHES || hybrid_range_dense_pays(rc.total, stored_bytes_, pass_bytes, nq, n))) {
            if (r8 && (!int_l2() || ensure_shadow(st))) {
                path = 2;
            } else if (r32 && ensure_shadow(st) && shadow_values_in_range()) {
                path = 1;
            }
        }
    }
    if (out_modes && path)
        for (size_t i = 0; i < nq; i++) out_modes[i] = HYBRID_BATCHES;
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_) dev_ctx_ = checkout();
    QueryCtx *c = dev_ctx_.get();
    if (!c) return -1;
    collect_dev_timing_locked();
    const CoarseKind kind = path == 1 ? CoarseF16 : CoarseDirect8;
    const CoarsePlan cp = path ? plan_coarse(v, nq32, kind, 1, 0, 1, 1, true) : CoarsePlan{};
    const size_t qpitch = query_pitch();
    const uint32_t words = path ? (uint32_t)((n + 31) / 32) : 0;
    // u32 words after the pinned table: 0, 1, .. nq - 1.  A dense route runs over the whole batch, so its positions are the queries
    // themselves
    std::vector<uint32_t> iota(nq);
    for (uint32_t i = 0; i < nq32; i++) iota[i] = i;
    const size_t tab_elems = ragged_table_elems(nq, nq);
    uint64_t *tab;
    uint32_t *d_total, *d_ok, *d_flags, *d_live, *bm;
    const uint32_t **d_live_ptr;
    RangeScratch rs;
    const auto layout = [&](void *base) {
        BatchScratch sc(base);
        tab = sc.take<uint64_t>(tab_elems);
        if (path) rs.take(sc, *this, kind, cp, nq32, false);
        d_total = sc.take<uint32_t>(1);
        d_ok = sc.take<uint32_t>(path ? nq : 0); // the route proved the query
        d_flags = sc.take<uint32_t>(nq);         // LastCoarseFlags
        d_live = sc.take<uint32_t>(path ? nq : 0);
        d_live_ptr = sc.take<const uint32_t *>(path ? nq : 0);
        bm = sc.take<uint32_t>((size_t)(path ? nq : 0) * words);
        return sc.words();
    };
    if (!c->need_cand(layout(nullptr))) return -1;
    layout(c->d_cand);
    RaggedBatch b;
    bool ok = true;
    if (!upload_ragged_table(tab, d_doc_ids, d_counts, caps, nq32, iota, st, b, ok)) return -1;
    const uint32_t *d_iota = reinterpret_cast<const uint32_t *>(tab + 4 * nq + 2);
    ok = ok && cudaMemsetAsync(d_counts_out, 0, nq * 4, st) == cudaSuccess;
    RaggedBatch bg = b; // the gather's batch: every query, or (dense route) the open ones
    LaunchCounters lc;
    uint64_t *comp = reinterpret_cast<uint64_t *>(d_labels);
    if (path) {
        // 1. row-space filter bitmaps; 2. range_device's route over the whole batch with them; 3. the open queries to the gather
        ok = ok && cudaMemsetAsync(bm, 0, (size_t)nq * words * 4, st) == cudaSuccess;
        ok = ok && launch_filter_bitmaps(b, d_iota, nq32, rc.max_cap, d_label_to_id_, (uint32_t)l2i_size_, bm, words, st, &lc) == cudaSuccess;
        ok = ok && enqueue_range_route(*c, v, kind, cp, rs, d_q, qpitch, nq32, d_radii, bm, words,
                                       RangeOut{comp, cap32, d_ok, d_counts_out, nullptr, d_total, nullptr}, st, lc);
        ok = ok && launch_hybrid_open(b, d_iota, d_ok, d_flags, d_live, d_live_ptr, st, &lc) == cudaSuccess;
        bg.counts = d_live_ptr;
    } else {
        ok = ok && cudaMemsetAsync(d_flags, 0, nq * 4, st) == cudaSuccess;
    }
    // after a dense route most chunks of the caps are empty: a grid of a few CTAs per SM strides over them
    const uint64_t max_grid = path ? (uint64_t)device_sm_count() * 16 : 0;
    ok = ok && launch_gather_ragged_range(v, d_q, qpitch, bg, tab + 3 * nq + 1, rc.blocks, d_label_to_id_, (uint32_t)l2i_size_,
                                          multi_ ? d_label_rows_ : nullptr, d_radii, cap32, comp, d_counts_out, st, &lc, max_grid) == cudaSuccess;
    ok = ok && launch_range_finish(d_labels, d_scores, d_counts_out, nq32, cap32, d_id_to_label_, order == BY_ID, st, &lc) == cudaSuccess;
    c->d_last_ok = d_flags;
    c->last_ok_n = nq32;
    last_batch_coarse_ = true; // LastCoarseFlags: 1 = a dense route answered the query, 0 = the gather
    last_batch_path_ = path;
    if (path) coarse_batches_++;
    dev_timing_pending_ = ok && path;
    dev_timing_bytes_ = path == 2 ? (uint64_t)n * dim_ : (uint64_t)n * dim_ * 2;
    launches_total_ += lc.launches;
    return ok ? 0 : -1;
}

// ------------------------------------------------------------------------------------------------
// request combiner for the stock single-query entry point (opt-in)
// ------------------------------------------------------------------------------------------------
struct FlatIndex::TopkReq {
    const void *blob;
    std::vector<size_t> labels;
    std::vector<double> scores;
    int code = VecSim_QueryReply_OK;
};

int FlatIndex::microbatch_window_us() {
    static int v = -1;
    if (v < 0) {
        const char *e = getenv("VECSIM_B200_MICROBATCH_US");
        v = e ? std::max(0, atoi(e)) : 0;
    }
    return v;
}

VecSimQueryReply *FlatIndex::topk_combined(const void *q, size_t k, VecSimQueryParams *qp, VecSimQueryReply_Order order) {
    const int window = microbatch_window_us();
    // only what the batched entry point serves in one pass; everything else keeps the direct route
    if (window <= 0 || multi_ || k == 0 || k > (size_t)kMaxFusedK || count_ < 65536) return topk(q, k, qp, order);
    // fp16 / bf16 corpora: a combined batch >= 16 would ride the tensor-core direct route, whose scores are within the 1e-2
    // bar but not bit-identical with the single-query scan — the answer would depend on how many callers were concurrent
    if (dtype_ == DT_F16 || dtype_ == DT_BF16) return topk(q, k, qp, order);
    void *tctx = qp ? qp->timeoutCtx : nullptr;
    auto *rep = new VecSimQueryReply();
    last_mode_ = STANDARD_KNN;
    if (timed_out(tctx)) {
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    using Batcher = MicroBatcher<TopkReq>;
    std::shared_ptr<void> holder;
    {
        std::lock_guard<std::mutex> g(mb_mu_);
        auto &slot = batchers_[k];
        if (!slot) {
            const size_t blob_bytes = dim_ * elem_bytes_;
            slot = std::shared_ptr<void>(
                new Batcher(256, std::chrono::microseconds(window),
                            [this, k, blob_bytes](std::vector<TopkReq *> &reqs) {
                                const size_t nq = reqs.size();
                                std::vector<uint8_t> blobs(nq * blob_bytes);
                                for (size_t i = 0; i < nq; i++) memcpy(blobs.data() + i * blob_bytes, reqs[i]->blob, blob_bytes);
                                std::vector<size_t> labels(nq * k);
                                std::vector<double> scores(nq * k);
                                const int code = topk_batch(blobs.data(), blob_bytes, nq, k, nullptr, labels.data(), scores.data());
                                for (size_t i = 0; i < nq; i++) {
                                    reqs[i]->code = code;
                                    reqs[i]->labels.assign(labels.begin() + i * k, labels.begin() + (i + 1) * k);
                                    reqs[i]->scores.assign(scores.begin() + i * k, scores.begin() + (i + 1) * k);
                                }
                            },
                            [](TopkReq &r) { r.code = -1; }),
                [](void *p) { delete static_cast<Batcher *>(p); });
        }
        holder = slot;
    }
    TopkReq r;
    r.blob = q;
    static_cast<Batcher *>(holder.get())->submit(r);
    if (r.code == VecSim_QueryReply_TimedOut || timed_out(tctx)) {
        rep->code = VecSim_QueryReply_TimedOut;
        return rep;
    }
    if (r.code != VecSim_QueryReply_OK) {
        log("warning", "vecsim_b200: combined top-k query failed on device");
        return rep;
    }
    for (size_t j = 0; j < k && j < r.labels.size(); j++)
        if (r.labels[j] != SIZE_MAX) rep->results.push_back({r.labels[j], r.scores[j]});
    finish_reply(rep, order);
    return rep;
}

// ------------------------------------------------------------------------------------------------
// info
// ------------------------------------------------------------------------------------------------
VecSimIndexBasicInfo FlatIndex::basic_info() const {
    VecSimIndexBasicInfo i{};
    i.algo = VecSimAlgo_BF;
    i.metric = metric_;
    i.type = type_;
    i.isMulti = multi_;
    i.isTiered = false;
    i.isDisk = false;
    i.blockSize = block_size_;
    i.dim = dim_;
    return i;
}
VecSimIndexStatsInfo FlatIndex::stats_info() const {
    VecSimIndexStatsInfo s{};
    s.memory = capacity_ * pitch_ + d_labels_cap_ * 8 + stage_cap_rows_ * pitch_ + id_to_label_.capacity() * sizeof(size_t) +
               (label_to_id_.size() + label_to_ids_.size()) * (sizeof(size_t) + sizeof(void *) * 2 + sizeof(idType));
    return s;
}

static const char *type_name(VecSimType t) {
    switch (t) {
    case VecSimType_FLOAT32: return "FLOAT32";
    case VecSimType_FLOAT64: return "FLOAT64";
    case VecSimType_BFLOAT16: return "BFLOAT16";
    case VecSimType_FLOAT16: return "FLOAT16";
    case VecSimType_INT8: return "INT8";
    case VecSimType_UINT8: return "UINT8";
    case VecSimType_INT32: return "INT32";
    default: return "INT64";
    }
}
static const char *mode_name(VecSearchMode m) { // vec_utils.cpp VecSimSearchMode_ToString
    switch (m) {
    case EMPTY_MODE: return "EMPTY_MODE";
    case STANDARD_KNN: return "STANDARD_KNN";
    case HYBRID_ADHOC_BF: return "HYBRID_ADHOC_BF";
    case HYBRID_BATCHES: return "HYBRID_BATCHES";
    case HYBRID_BATCHES_TO_ADHOC_BF: return "HYBRID_BATCHES_TO_ADHOC_BF";
    default: return "RANGE_QUERY";
    }
}

VecSimIndexDebugInfo FlatIndex::debug_info() const {
    VecSimIndexDebugInfo info;
    memset(&info, 0, sizeof(info));
    info.commonInfo.basicInfo = basic_info();
    info.commonInfo.indexSize = count_;
    info.commonInfo.indexLabelCount = multi_ ? label_to_ids_.size() : label_to_id_.size();
    info.commonInfo.memory = stats_info().memory;
    info.commonInfo.lastMode = last_mode_;
    info.bfInfo.dummy = 0;
    return info;
}

VecSimDebugInfoIterator *FlatIndex::debug_iterator() const {
    auto *it = new VecSimDebugInfoIterator();
    auto str = [&](const char *name, const char *v) {
        VecSim_InfoField f{};
        f.fieldName = name;
        f.fieldType = INFOFIELD_STRING;
        f.fieldValue.stringValue = v;
        it->fields.push_back(f);
    };
    auto u64 = [&](const char *name, uint64_t v) {
        VecSim_InfoField f{};
        f.fieldName = name;
        f.fieldType = INFOFIELD_UINT64;
        f.fieldValue.uintegerValue = v;
        it->fields.push_back(f);
    };
    // order and names: brute_force.h:327-365 + vec_sim_index.h addCommonInfoToIterator
    str("ALGORITHM", "FLAT");
    str("TYPE", type_name(type_));
    u64("DIMENSION", dim_);
    str("METRIC", metric_ == VecSimMetric_L2 ? "L2" : metric_ == VecSimMetric_IP ? "IP" : "COSINE");
    u64("IS_MULTI_VALUE", multi_);
    u64("IS_DISK", 0);
    u64("INDEX_SIZE", count_);
    u64("INDEX_LABEL_COUNT", multi_ ? label_to_ids_.size() : label_to_id_.size());
    u64("MEMORY", stats_info().memory);
    str("LAST_SEARCH_MODE", mode_name(last_mode_));
    u64("BLOCK_SIZE", block_size_);
    return it;
}

int FlatIndex::last_coarse_flags(uint32_t *out, size_t n) {
    std::lock_guard<std::mutex> dg(dev_mu_);
    if (!dev_ctx_ || !last_batch_coarse_ || !dev_ctx_->d_last_ok || dev_ctx_->last_ok_n < n) return -1;
    if (cudaDeviceSynchronize() != cudaSuccess) return -1;
    return cudaMemcpy(out, dev_ctx_->d_last_ok, n * 4, cudaMemcpyDeviceToHost) == cudaSuccess ? 0 : -1;
}

void set_coarse_mode(int mode) { g_coarse_mode.store(mode); }

// dev_mu_ held.  Folds the CUDA-event timing of the last topk_batch_device scan into the stats.
void FlatIndex::collect_dev_timing_locked() {
    if (!dev_timing_pending_ || !dev_ctx_) return;
    if (cudaEventSynchronize(dev_ctx_->ev_stop) == cudaSuccess) record_scan(dev_ctx_.get(), dev_timing_bytes_);
    dev_timing_pending_ = false;
}

VecSimB200_Stats FlatIndex::get_stats(bool reset) {
    {
        std::lock_guard<std::mutex> dg(dev_mu_);
        collect_dev_timing_locked();
    }
    std::lock_guard<std::mutex> g(stats_mu_);
    VecSimB200_Stats s{};
    s.kernel_launches = launches_total_.load();
    s.scan_launches = scan_launches_;
    s.scan_device_us = scan_us_;
    s.scan_bytes = scan_bytes_;
    if (reset) {
        launches_total_ = 0;
        scan_launches_ = 0;
        scan_us_ = 0;
        scan_bytes_ = 0;
    }
    return s;
}

} // namespace rsb200
