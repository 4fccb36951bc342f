// trn_ctx: the device-resident index source + batch executor behind the C ABI (include/trinity_b200.h).
// Host responsibilities mirror the host side of the reference's exec path:
//   * upload == AccessProxy construction + Decoder::init for every term (google_codec.cpp:936-983, lucene_codec.cpp:877-932)
//   * plan compile == queryexec_ctx::build_iterator + build_span (exec.cpp:253-505): planner.h (plan_batch), called per batch here
// There is NO CPU execution fallback: every docset/score operation runs in kernels.cu.
#include "../../include/trinity_b200.h"
#include "codecs.h"
#include "device_types.h"
#include "hitcursor.h"
#include "chunkplan.h"
#include "isectplan.h"
#include "percplan.h"
#include "mergeplan.h"
#include "kernels.h"
#include "planner.h"
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <thread>
#include <utility>
#include <vector>

using namespace trn;

namespace {
// Device memory (DevBuf) or pinned host memory (PinBuf) that frees itself when it goes out of scope.  It moves but does not copy, so
// every allocation has exactly one owner.  release() frees early, where a caller lowers its peak memory.
template <bool Pinned> struct Buf {
        void * p{nullptr};
        size_t cap{0};
        Buf() = default;
        Buf(Buf &&o) noexcept : p(std::exchange(o.p, nullptr)), cap(std::exchange(o.cap, 0)) {} // (declaring the moves deletes the copies)
        Buf &operator=(Buf &&o) noexcept {
                if (this != &o) {
                        release();
                        std::swap(p, o.p);
                        std::swap(cap, o.cap);
                }
                return *this;
        }
        ~Buf() {
                release();
        }
        // at least `bytes`; the contents are not kept
        cudaError_t ensure(size_t bytes) {
                if (bytes <= cap)
                        return cudaSuccess;
                release();
                size_t      want = bytes + bytes / 8 + 256;
                cudaError_t e    = Pinned ? cudaHostAlloc(&p, want, cudaHostAllocDefault) : cudaMalloc(&p, want);
                if (e == cudaSuccess)
                        cap = want;
                return e;
        }
        // at least `need`, keeping the first `keep` bytes: they are copied once the copies queued on `s` have landed.  On failure the
        // buffer is unchanged.
        cudaError_t grow(size_t need, size_t keep, cudaStream_t s) {
                static_assert(Pinned, "the old contents are copied on the host");
                if (need <= cap)
                        return cudaSuccess;
                void *       np{nullptr};
                const size_t want = need + need / 4 + 4096;
                if (const cudaError_t e = cudaHostAlloc(&np, want, cudaHostAllocDefault); e != cudaSuccess)
                        return e;
                if (p && keep) {
                        cudaStreamSynchronize(s);
                        std::memcpy(np, p, keep);
                }
                release();
                p   = np;
                cap = want;
                return cudaSuccess;
        }
        void release() {
                if (p) {
                        if constexpr (Pinned)
                                cudaFreeHost(p);
                        else
                                cudaFree(p);
                }
                p   = nullptr;
                cap = 0;
        }
        template <class T> T *as() const {
                return static_cast<T *>(p);
        }
};
using DevBuf = Buf<false>;
using PinBuf = Buf<true>;

// A CUDA event or stream the context created and destroys (null until created).  It converts to the handle the runtime calls take.
template <class H, cudaError_t (*Destroy)(H)> struct Owned {
        H h{nullptr};
        Owned() = default;
        Owned(const Owned &)            = delete;
        Owned &operator=(const Owned &) = delete;
        ~Owned() {
                if (h)
                        Destroy(h);
        }
        operator H() const {
                return h;
        }
};
using Event  = Owned<cudaEvent_t, cudaEventDestroy>;
using Stream = Owned<cudaStream_t, cudaStreamDestroy>;
} // namespace

struct trn_ctx {
        int          device{0};
        cudaStream_t stream{nullptr};
        std::string  err;
        int          num_sms{132}; // set from the device in trn_create
        // index
        bool                 have_index{false};
        PlanConfig           pc; // the planner's view of the index, its knobs and the kernels' limits (trn_create, trn_upload_index)
        uint32_t             block_docs{32}; // documents per full block of the uploaded index (GOOGLE 32 unless built for the decode sweep; LUCENE 128)
        uint32_t             nterms{0}, ntiles{0}; // ntiles: of pc.tile_shift
        int                  flat_threads{320}; // TRN_SF_THREADS: CTA size of k_score_flat (320: two CTAs per SM; 512: one; any other value runs 320)
        uint64_t             index_bytes{0}, dir_bytes{0}, total_blocks{0}, total_postings{0};
        DevBuf               d_index, d_blk_last, d_blk_off, d_terms, d_tile_first, d_masked;
        bool                 have_masked{false};
        // per-query document filters (trn_docset_create): handle = (epoch & 0xffff) << 16 | slot; a new upload frees every set and bumps the epoch
        struct DocSet {
                DevBuf   bits;       // laid out like d_masked
                uint32_t lo{1}, hi{0}; // first and last docID (lo > hi: empty)
                bool     live{false};
        };
        std::vector<DocSet> docsets;
        uint32_t            docset_epoch{0};
        uint32_t            docset_max{0xffffu}; // TRN_DOCSET_MAX: sets a context holds at once (at most 65535)
        DevBuf              d_filters;           // the batch's DevFilter per query (exec_device_impl, filtered batches only)
        DevBuf               d_dense, d_dense_off; // resident bitmaps of the dense terms (select_dense_terms) and each term's first word in them
        uint32_t             dense_terms{0};       // terms with a bitmap (0: none, d_dense unused)
        uint64_t             dense_bytes{0};
        std::vector<uint32_t> h_dense_off;          // host copy of d_dense_off (trn_debug_dense_bitmap)
        DevBuf               d_probe_off;          // per term its first word in d_dense for the candidate-driven probes (select_probe_terms)
        uint32_t             probe_terms{0};       // terms of the probe tier, laid out in d_dense behind the dense bitmaps
        uint64_t             probe_bytes{0};
        std::vector<DevTerm> h_terms;
        GroupStarts          h_groups; // GOOGLE: the first docID of every 32-block group of every term (orders BatchPlan::cand_runs)
        // batch scratch (grow-only)
        DevBuf d_queries, d_steps, d_dense_runs, d_mixed_runs, d_cand_order, d_small[2], d_item_off, d_item_cnt, d_item_dst, d_seg_docids, d_seg_scores, d_out_docids[2], d_out_scores[2], d_q_offsets[2], d_cand,
            d_topk_docids, d_topk_scores, d_topk_counts, d_fq, d_leaves, d_luts, d_dec_units, d_dec_c, d_dec_docids, d_dec_freqs, d_dec_sums;
        PinBuf h_offsets, h_docids, h_scores, h_counts, h_small, h_chunk, h_item_desc;
        DevBuf d_hits, d_hit_base, d_hblk_off, d_hit_term; // LUCENE positions (trn_upload_hits)
        bool   have_hits{false};
        BlockDirectory              h_dir;     // LUCENE: kept for trn_upload_hits (the hits directory is laid out like the block directory)
        std::vector<term_index_ctx> h_termctx; // ...
        DevBuf d_item_desc[2];                 // compact results: per work item, matches | encoding << 30 (double-buffered like the outputs)
        std::vector<trn_qitems> qitems_set[2]; // compact results: the per-query item ranges of the last exec_device_impl call of each set
        std::vector<trn_qitems> h_qitems;      // ... of the whole batch, item_base rebased (what trn_result::qitems points to)
        std::vector<std::vector<trn_qitems>> qitems_chunk; // pipelined call: per chunk, until its results have been queued for the copy
        uint64_t                last_items_hint{0};
        Event ev0, ev1, evk0, evk1;
        bool  have_kernel_events{false};
        // pipelined host-buffer path (trn_exec_batch): kernels of chunk i+1 overlap the D2H of chunk i
        Stream       copy_stream;
        Event        ev_done[2], ev_d2h[2], ev_ck0[16], ev_ck1[16];
        uint64_t     chunk_postings{1000000000ull}; // TRN_CHUNK_POSTINGS: referenced postings a pipeline chunk must carry (~1.1 ms of k_exec_docs)
        bool         taper_chunks{true};             // TRN_TAPER_CHUNKS=0: equal chunks only
        bool         chunk_rule_sqrt{true};          // TRN_CHUNK_RULE=postings: chunk count from the referenced postings alone
        double       chunk_tail_ms{0.15}, chunk_tail_tree_ms{0.9}; // TRN_CHUNK_TAIL_US / TRN_CHUNK_TAIL_TREE_US: modelled cost of one more launch
        uint64_t     hint_bytes{0}, hint_postings{0}; // result bytes / referenced postings of the previous host-buffer batch ...
        uint32_t     hint_nq{0};                     // ... and its shape: the next batch of the same shape sizes its chunks from them
        int          hint_mode{-1};
        uint32_t     pipeline_chunks{8}; // TRN_PIPELINE_CHUNKS: upper bound of the chunk plan (chunkplan.h)
        uint32_t     last_items{0}; // work items of the last exec_device_impl call (compact results: entries of item_desc)
        uint64_t     last_total_hint{0};
        // host-side breakdown of the last trn_exec_batch / trn_exec_batch_device call (trn_last_timings)
        trn_timings tm{};
        // last batch
        int      last_mode{-1};
        uint32_t last_nq{0}, last_k{0}, last_launches{0};
        uint64_t last_postings{0}, last_bytes{0};
        std::vector<uint8_t> last_routes; // TRN_ROUTE_* of every query of the last batch (trn_debug_last_routes)
        // the default exec mode (trn_exec_matches): collect programs, per-chunk intermediates and outputs, the pinned result
        struct MatchBufs {
                DevBuf d_cq, d_cterms, d_cphrases, d_cargs, d_cprog, d_mask, d_nterms, d_nhits, d_tscan, d_hscan, d_part, d_term_off, d_terms, d_freqs,
                    d_hit_off, d_hits, d_error;
                PinBuf h_doc_off, h_docids, h_term_off, h_terms, h_freqs, h_hit_off, h_hits, h_small;
                Event  ev_docs, ev_c0, ev_c1, ev_w0, ev_w1, ev_end;
        } mt;
        uint64_t match_chunk{1ull << 22}; // TRN_MATCH_CHUNK: matches per chunk of the write pass (halved while its outputs do not fit)
        // query-token intersections (trn_intersect): device scratch of both passes, the result
        struct IsectBufs {
                DevBuf d_reqs, d_tok, d_small, d_keys, d_first, d_tile_last, d_carry, d_base, d_cmask, d_cfirst, d_estart, d_eoff, d_smask, d_sslot, d_counts;
                std::vector<uint64_t> offsets, masks;
                std::vector<uint32_t> counts;
                Event                 ev[4];
        } it;
        uint32_t isect_max_masks{kIsectMaxMasks}; // TRN_ISECT_MAX_MASKS: distinct masks a request may have (lowers the limit only)
        uint64_t perc_max_ids{0xFFFFFFFFull};      // TRN_PERC_MAX_IDS: ids a registry may issue (lowers the limit only)
        uint64_t perc_max_entries{1ull << 32};     // TRN_PERC_MAX_ENTRIES: anchor entries a registry may hold (lowers the limit only)
        // percolator (trn_percolator_register / trn_percolate): the registry, the batch scratch, the pinned result
        struct PercBufs {
                bool                have{false};
                uint32_t            next_id{0}, nterms{0}, nunanchored{0}; // next_id: ids issued since the registration (removed ones included)
                trn_percolator_info info{};
                DevBuf d_queries, d_ops, d_pterms, d_covers, d_csr_off, d_csr, d_unanch; // the registry
                // the host's view of the registry for trn_percolator_add / trn_percolator_remove
                struct Sizes {
                        uint32_t nops, npt, ncover;
                        uint8_t  status;
                };
                std::vector<Sizes>    sizes;     // per issued id
                std::vector<uint32_t> removed;   // bitmap over the issued ids
                std::vector<uint32_t> term_cost; // the registration's (empty: all equal)
                uint32_t              nlive{0}, nnever{0};
                uint64_t              nentries{0};                              // entries of d_csr
                uint64_t              ops_used{0}, pt_used{0}, cov_used{0};     // entries of d_ops / d_pterms / d_covers in use ...
                uint64_t              dead_words{0};                            // ... and the words of removed queries among them
                DevBuf d_removed, d_keep, d_kscan, d_upart, d_cnt, d_toff, d_new, d_new_terms, d_new_unanch; // update scratch (grow-only)
                Event  uev[2];
                float  update_ms{0}, update_host_ms{0}; // the last add / remove: CUDA-event time of its device work, host time
                DevBuf d_doc_off, d_tokens, d_docs, d_counts, d_small, d_part, d_out_off, d_out, d_bitmaps, d_dense_slot;
                PinBuf h_offsets, h_ids;
                Event  ev[4];
        } pq;
        // indexer (trn_index_documents): the last result (its working memory lives for one call only)
        struct IndexBufs {
                std::vector<uint8_t>  index, hits;
                std::vector<trn_term> terms;
                Event                 ev[5];
        } ix;
        // merge (trn_merge_sources): the last result
        struct MergeBufs {
                std::vector<uint8_t>  index, hits;
                std::vector<trn_term> terms;
                std::vector<uint32_t> term_source, term_index;
                Event                 ev[8];
        } mg;
};

#define CK(call)                                                                                                                                               \
        do {                                                                                                                                                   \
                cudaError_t e__ = (call);                                                                                                                      \
                if (e__ != cudaSuccess) {                                                                                                                      \
                        c->err = std::string(#call) + ": " + cudaGetErrorString(e__);                                                                          \
                        return TRN_ERR_CUDA;                                                                                                                   \
                }                                                                                                                                              \
        } while (0)

static inline double now_ms() {
        return std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

static DevIndex dev_index(trn_ctx *c);

static int fail(trn_ctx *c, int code, const std::string &m) {
        c->err = m;
        return code;
}

// the planner's configuration as a new context starts with it: the knobs from the environment, the limits of this build's kernels
static PlanConfig initial_plan_config() {
        PlanConfig pc            = plan_config_from_env();
        pc.score_flat_max_leaves = score_flat_max_leaves();
        pc.docs_stage_bytes      = exec_docs_stage_bytes();
        pc.cand_smem_bytes[0]    = exec_docs_cand_smem_bytes(false);
        pc.cand_smem_bytes[1]    = exec_docs_cand_smem_bytes(true);
        pc.mixed_smem_bytes      = exec_docs_mixed_smem_bytes();
        return pc;
}

// =================================================================================================== C ABI: lifecycle
extern "C" int trn_create(int device, trn_ctx **out) {
        if (!out)
                return TRN_ERR_ARG;
        auto c    = new trn_ctx();
        c->device = device;
        *out      = c;
        int ndev{0};
        cudaError_t e = cudaGetDeviceCount(&ndev);
        if (e != cudaSuccess || device < 0 || device >= ndev) {
                // No silent CPU fallback: the context is unusable without a CUDA device.
                c->err = std::string("trn_create: no usable CUDA device (") + (e != cudaSuccess ? cudaGetErrorString(e) : "device index out of range") + ")";
                return TRN_ERR_CUDA;
        }
        CK(cudaSetDevice(device));
        cudaDeviceProp prop;
        CK(cudaGetDeviceProperties(&prop, device));
        c->num_sms = prop.multiProcessorCount;
        c->pc      = initial_plan_config();
        if (const char *e = getenv("TRN_SF_THREADS"))
                c->flat_threads = atoi(e);
        if (const char *e = getenv("TRN_PIPELINE_CHUNKS")) {
                const int v = atoi(e);
                if (v >= 1 && v <= 16)
                        c->pipeline_chunks = uint32_t(v);
        }
        if (const char *e = getenv("TRN_TAPER_CHUNKS"))
                c->taper_chunks = atoi(e) != 0;
        if (const char *e = getenv("TRN_CHUNK_RULE"))
                c->chunk_rule_sqrt = std::string(e) != "postings";
        if (const char *e = getenv("TRN_CHUNK_TAIL_US"))
                c->chunk_tail_ms = std::max(1.0, atof(e)) / 1000.0;
        if (const char *e = getenv("TRN_CHUNK_TAIL_TREE_US"))
                c->chunk_tail_tree_ms = std::max(1.0, atof(e)) / 1000.0;
        if (const char *e = getenv("TRN_CHUNK_POSTINGS")) {
                const long long v = atoll(e);
                if (v >= 1)
                        c->chunk_postings = uint64_t(v);
        }
        if (const char *e = getenv("TRN_MATCH_CHUNK")) {
                const long long v = atoll(e);
                if (v >= 1)
                        c->match_chunk = uint64_t(v);
        }
        if (const char *e = getenv("TRN_DOCSET_MAX")) {
                const long long v = atoll(e);
                if (v >= 0 && v < 0xffffll)
                        c->docset_max = uint32_t(v);
        }
        if (const char *e = getenv("TRN_ISECT_MAX_MASKS")) {
                const long long v = atoll(e);
                if (v >= 1 && v < (long long)kIsectMaxMasks)
                        c->isect_max_masks = uint32_t(v);
        }
        if (const char *e = getenv("TRN_PERC_MAX_IDS")) {
                const long long v = atoll(e);
                if (v >= 1 && uint64_t(v) < c->perc_max_ids)
                        c->perc_max_ids = uint64_t(v);
        }
        if (const char *e = getenv("TRN_PERC_MAX_ENTRIES")) {
                const long long v = atoll(e);
                if (v >= 1 && uint64_t(v) < c->perc_max_entries)
                        c->perc_max_entries = uint64_t(v);
        }
        CK(cudaStreamCreateWithFlags(&c->copy_stream.h, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
                CK(cudaEventCreateWithFlags(&c->ev_done[i].h, cudaEventDisableTiming));
                CK(cudaEventCreateWithFlags(&c->ev_d2h[i].h, cudaEventDisableTiming));
        }
        for (int i = 0; i < 16; ++i) {
                CK(cudaEventCreate(&c->ev_ck0[i].h));
                CK(cudaEventCreate(&c->ev_ck1[i].h));
        }
        CK(cudaEventCreate(&c->ev0.h));
        CK(cudaEventCreate(&c->ev1.h));
        CK(cudaEventCreate(&c->evk0.h));
        CK(cudaEventCreate(&c->evk1.h));
        return TRN_OK;
}

extern "C" void trn_destroy(trn_ctx *c) {
        if (!c)
                return;
        cudaSetDevice(c->device);
        delete c;
}

extern "C" const char *trn_last_error(trn_ctx *c) {
        return c ? c->err.c_str() : "null ctx";
}

extern "C" int trn_set_stream(trn_ctx *c, void *s) {
        if (!c)
                return TRN_ERR_ARG;
        c->stream = static_cast<cudaStream_t>(s);
        return TRN_OK;
}

// =================================================================================================== upload
// The resident docID bitmaps of the index just copied, both tiers (select_dense_terms, select_probe_terms) in one array, built on the
// device from the doc-delta sections: exact copies of the terms' docID sets, like the block directory.  Not being able to allocate them
// does not fail the upload: the probe tier goes first and the dense tier keeps its bitmaps if they alone fit; without either the source
// runs without bitmaps.  trn_last_error says why.
static int upload_dense(trn_ctx *c) {
        c->dense_terms = 0;
        c->dense_bytes = 0;
        c->probe_terms = 0;
        c->probe_bytes = 0;
        c->h_dense_off.clear();
        DenseSelection s, p; // p.off: what d_probe_off holds
        try {
                s = select_dense_terms(c->pc, c->h_terms, c->index_bytes);
                p = select_probe_terms(c->pc, c->h_terms, c->index_bytes, s);
        } catch (const std::bad_alloc &) {
                s = p = DenseSelection{};
                c->err = "dense-term bitmaps off for this index: out of host memory";
        }
        // k_build_dense reads blocks of the format's 32 documents; an index built with another block size (decode sweep) gets no
        // bitmaps, and the exec entry points refuse it
        if (c->block_docs != Codecs::Google::N)
                s = p = DenseSelection{};
        DevBuf      sel, pre;
        cudaError_t e = cudaSuccess;
        auto        allocate = [&] {
                const size_t nsel = s.order.size() + p.order.size();
                e                 = c->d_dense.ensure((s.words + p.words) * 4);
                if (e == cudaSuccess)
                        e = c->d_dense_off.ensure(std::max<size_t>(4, s.off.size() * 4));
                if (e == cudaSuccess)
                        e = c->d_probe_off.ensure(std::max<size_t>(4, p.off.size() * 4));
                if (e == cudaSuccess)
                        e = sel.ensure(nsel * 4);
                if (e == cudaSuccess)
                        e = pre.ensure((nsel + 1) * 8);
                if (e != cudaSuccess) {
                        (void)cudaGetLastError(); // an allocation failure is not sticky: clear it
                        for (DevBuf *b : {&c->d_dense, &c->d_dense_off, &c->d_probe_off, &sel, &pre})
                                b->release();
                }
        };
        if (!p.order.empty()) {
                allocate();
                if (e != cudaSuccess) {
                        c->err          = std::string("probe bitmaps off for this index: ") + cudaGetErrorString(e);
                        p.order.clear();
                        p.words         = 0;
                        p.off           = s.off;
                        e               = cudaSuccess;
                }
        }
        if (p.order.empty() && !s.order.empty()) {
                allocate();
                if (e != cudaSuccess)
                        c->err = std::string("dense-term bitmaps off for this index: ") + cudaGetErrorString(e);
        }
        std::vector<uint32_t>           order;
        std::vector<unsigned long long> prefix;
        if (e == cudaSuccess) {
                try {
                        order = s.order;
                        order.insert(order.end(), p.order.begin(), p.order.end());
                        prefix.assign(order.size() + 1, 0ull);
                        for (size_t i = 0; i < order.size(); ++i)
                                prefix[i + 1] = prefix[i] + c->h_terms[order[i]].nblocks;
                } catch (const std::bad_alloc &) {
                        order.clear();
                        c->err = "dense-term bitmaps off for this index: out of host memory";
                }
        }
        if (order.empty()) {
                c->d_dense.release();
                c->d_dense_off.release();
                c->d_probe_off.release();
                return TRN_OK;
        }
        CK(cudaMemsetAsync(c->d_dense.p, 0, (s.words + p.words) * 4, c->stream));
        CK(cudaMemcpyAsync(c->d_dense_off.p, s.off.data(), s.off.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->d_probe_off.p, p.off.data(), p.off.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(sel.p, order.data(), order.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(pre.p, prefix.data(), prefix.size() * 8, cudaMemcpyHostToDevice, c->stream));
        c->dense_terms = uint32_t(s.order.size()); // dev_index hands the bitmaps out from here on
        c->probe_terms = uint32_t(p.order.size());
        // the launch check reads the thread's last error: drop one a failed call elsewhere left behind (e.g. trn_destroy's cudaSetDevice
        // of a context created for a device that does not exist)
        (void)cudaGetLastError();
        const cudaError_t le = launch_build_dense(dev_index(c), sel.as<uint32_t>(), pre.as<unsigned long long>(), uint32_t(order.size()), prefix.back(),
                                                  c->d_dense.as<uint32_t>(), c->stream);
        const cudaError_t se = cudaStreamSynchronize(c->stream);
        if (le != cudaSuccess || se != cudaSuccess) {
                c->dense_terms = 0;
                c->probe_terms = 0;
                return fail(c, TRN_ERR_CUDA, std::string("building the dense-term bitmaps: ") + cudaGetErrorString(le != cudaSuccess ? le : se));
        }
        c->dense_bytes = s.words * 4;
        c->probe_bytes = p.words * 4;
        c->h_dense_off = std::move(s.off);
        return TRN_OK;
}

// every docID set of the context is dropped: its handles become stale (trn_upload_index; the sets' sizes follow the old max_docid)
static void drop_docsets(trn_ctx *c) {
        c->docsets.clear();
        ++c->docset_epoch;
}

extern "C" int trn_upload_index(trn_ctx *c, int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid) {
        if (!c || !index || !terms || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return c ? fail(c, TRN_ERR_ARG, "trn_upload_index: bad arguments") : TRN_ERR_ARG;
        if (nbytes >= (1ull << 32))
                return fail(c, TRN_ERR_ARG, "index larger than 4 GiB: one IndexSource is limited to range32_t offsets (codecs.h:17-55); shard it");
        CK(cudaSetDevice(c->device));
        BlockDirectory       dir;
        std::vector<DevTerm> ht;
        try {
                const int threads = int(std::max(1u, std::min(64u, std::thread::hardware_concurrency())));
                build_directory(codec, index, nbytes, terms, nterms, threads, dir);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_index: out of host memory while building the block directory");
        } catch (const std::exception &e) {
                return fail(c, TRN_ERR_FORMAT, e.what());
        }
        GroupStarts gs;
        try {
                ht = dev_terms(dir, terms, nterms);
                if (codec == TRN_CODEC_GOOGLE)
                        gs = group_starts(dir);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_index: out of host memory");
        }
        uint32_t min_docid;
        docid_span(ht, min_docid, max_docid);
        c->have_index   = false; // until the new index is completely in place
        drop_docsets(c);
        c->pc.codec     = codec;
        c->pc.min_docid = min_docid;
        c->pc.max_docid = max_docid;
        c->block_docs   = dir.block_docs;
        c->nterms       = nterms;
        const uint32_t W = 1u << c->pc.tile_shift;
        c->ntiles       = uint32_t((uint64_t(max_docid) + 1 + W - 1) >> c->pc.tile_shift);
        c->h_terms      = std::move(ht);
        c->h_groups     = std::move(gs);
        c->total_blocks   = 0;
        c->total_postings = 0;
        for (const auto &d : c->h_terms) {
                c->total_blocks += d.nblocks;
                c->total_postings += d.documents;
                if (d.nblocks && d.last_doc > max_docid)
                        return fail(c, TRN_ERR_ARG, "a term holds a docID above max_docid");
        }
        CK(c->d_index.ensure(nbytes + 256));
        CK(cudaMemsetAsync(c->d_index.p, 0, nbytes + 256, c->stream));
        CK(cudaMemcpyAsync(c->d_index.p, index, nbytes, cudaMemcpyHostToDevice, c->stream));
        const size_t nent = dir.blk_last.size();
        CK(c->d_blk_last.ensure(std::max<size_t>(4, nent * 4)));
        CK(c->d_blk_off.ensure(std::max<size_t>(4, nent * 4)));
        CK(cudaMemcpyAsync(c->d_blk_last.p, dir.blk_last.data(), nent * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->d_blk_off.p, dir.blk_off.data(), nent * 4, cudaMemcpyHostToDevice, c->stream));
        CK(c->d_terms.ensure(std::max<size_t>(4, nterms * sizeof(DevTerm))));
        CK(cudaMemcpyAsync(c->d_terms.p, c->h_terms.data(), nterms * sizeof(DevTerm), cudaMemcpyHostToDevice, c->stream));
        CK(c->d_tile_first.ensure(std::max<size_t>(4, dir.tile_first.size() * 4)));
        if (!dir.tile_first.empty())
                CK(cudaMemcpyAsync(c->d_tile_first.p, dir.tile_first.data(), dir.tile_first.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->index_bytes = nbytes;
        c->dir_bytes   = dir.bytes();
        if (const int rc = upload_dense(c); rc != TRN_OK)
                return rc;
        c->have_index  = true;
        c->have_hits   = false; // positions belong to the index they were uploaded for
        c->h_dir       = BlockDirectory{};
        c->h_termctx.clear();
        if (codec == TRN_CODEC_LUCENE) {
                try {
                        c->h_termctx.resize(nterms);
                        for (uint32_t i = 0; i < nterms; ++i) {
                                c->h_termctx[i].documents = terms[i].documents;
                                c->h_termctx[i].offset    = terms[i].chunk_off;
                                c->h_termctx[i].size      = terms[i].chunk_len;
                        }
                        dir.tile_first.clear();
                        dir.tile_first.shrink_to_fit();
                        c->h_dir = std::move(dir);
                } catch (const std::bad_alloc &) {
                        c->h_termctx.clear(); // trn_upload_hits will say so
                }
        }
        // the masked-documents bitmap belongs to the index it was set for (its size follows that index's max_docid): a new upload
        // starts with an empty registry, callers set it again (trn_set_masked_documents)
        c->have_masked = false;
        return TRN_OK;
}


// LUCENE positions: hits.data of the uploaded index (lucene_codec.cpp:401-513).  `index` = the bytes trn_upload_index received (they are
// read again on the host: the freqs give every block's first hit number); without this call phrase plans on a LUCENE source are refused.
extern "C" int trn_upload_hits(trn_ctx *c, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hbytes) {
        if (!c || !index || (!hits && hbytes))
                return c ? fail(c, TRN_ERR_ARG, "trn_upload_hits: bad arguments") : TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (c->pc.codec != TRN_CODEC_LUCENE)
                return fail(c, TRN_ERR_ARG, "trn_upload_hits: the GOOGLE codec keeps its hits inline (nothing to upload)");
        if (nbytes != c->index_bytes || c->h_termctx.size() != c->nterms)
                return fail(c, TRN_ERR_ARG, "trn_upload_hits: not the index this context holds");
        if (hbytes >= (1ull << 32))
                return fail(c, TRN_ERR_ARG, "hits.data larger than 4 GiB");
        CK(cudaSetDevice(c->device));
        HitsDirectory hd;
        try {
                const int threads = int(std::max(1u, std::min(64u, std::thread::hardware_concurrency())));
                build_hits_directory(index, nbytes, hits, hbytes, c->h_termctx.data(), c->nterms, c->h_dir, threads, hd);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_hits: out of host memory");
        } catch (const std::exception &e) {
                return fail(c, TRN_ERR_FORMAT, e.what());
        }
        std::vector<HitTerm> ht(c->nterms);
        for (uint32_t i = 0; i < c->nterms; ++i)
                ht[i] = HitTerm{hd.hb_begin[i], hd.sum_hits[i]};
        c->have_hits = false;
        CK(c->d_hits.ensure(hbytes + 256));
        CK(cudaMemsetAsync(c->d_hits.p, 0, hbytes + 256, c->stream));
        if (hbytes)
                CK(cudaMemcpyAsync(c->d_hits.p, hits, hbytes, cudaMemcpyHostToDevice, c->stream));
        CK(c->d_hit_base.ensure(std::max<size_t>(4, hd.hit_base.size() * 4)));
        CK(c->d_hblk_off.ensure(std::max<size_t>(4, hd.hblk_off.size() * 4)));
        CK(c->d_hit_term.ensure(std::max<size_t>(8, ht.size() * 8)));
        if (!hd.hit_base.empty())
                CK(cudaMemcpyAsync(c->d_hit_base.p, hd.hit_base.data(), hd.hit_base.size() * 4, cudaMemcpyHostToDevice, c->stream));
        if (!hd.hblk_off.empty())
                CK(cudaMemcpyAsync(c->d_hblk_off.p, hd.hblk_off.data(), hd.hblk_off.size() * 4, cudaMemcpyHostToDevice, c->stream));
        if (!ht.empty())
                CK(cudaMemcpyAsync(c->d_hit_term.p, ht.data(), ht.size() * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->have_hits = true;
        return TRN_OK;
}

extern "C" int trn_set_masked_documents(trn_ctx *c, const uint32_t *docids, uint64_t n) {
        if (!c)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (n && !docids)
                return fail(c, TRN_ERR_ARG, "trn_set_masked_documents: null docids");
        CK(cudaSetDevice(c->device));
        if (n == 0) {
                c->have_masked = false;
                return TRN_OK;
        }
        // one bit per docID, padded so that every (largest) tile can read its whole word range
        const uint64_t        span  = ((uint64_t(c->pc.max_docid) >> 17) + 2) << 17;
        std::vector<uint32_t> words(span / 32, 0u);
        for (uint64_t i = 0; i < n; ++i) {
                if (docids[i] == 0)
                        return fail(c, TRN_ERR_ARG, "masked docID 0 is not a document");
                if (docids[i] > c->pc.max_docid)
                        continue; // a newer source may mask documents this source never held
                words[docids[i] >> 5] |= 1u << (docids[i] & 31u);
        }
        CK(c->d_masked.ensure(words.size() * 4));
        CK(cudaMemcpyAsync(c->d_masked.p, words.data(), words.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->have_masked = true;
        return TRN_OK;
}

// ============================================================================================ per-query document filters
extern "C" int trn_docset_create(trn_ctx *c, const uint32_t *docids, uint64_t n, uint32_t *handle) {
        if (!c)
                return TRN_ERR_ARG;
        if (!handle || (n && !docids))
                return fail(c, TRN_ERR_ARG, "trn_docset_create: null argument");
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        CK(cudaSetDevice(c->device));
        uint32_t slot = 0, nlive = 0;
        while (slot < c->docsets.size() && c->docsets[slot].live)
                ++slot;
        for (const auto &d : c->docsets)
                nlive += d.live ? 1u : 0u;
        if (nlive >= c->docset_max)
                return fail(c, TRN_ERR_CAPACITY, "trn_docset_create: the context holds " + std::to_string(nlive) + " docID sets (TRN_DOCSET_MAX); destroy some");
        // the layout of trn_set_masked_documents: one bit per docID, padded so that every (largest) tile can read its whole word range
        const uint64_t        span = ((uint64_t(c->pc.max_docid) >> 17) + 2) << 17;
        std::vector<uint32_t> words;
        try {
                words.assign(span / 32, 0u);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_docset_create: out of host memory");
        }
        uint32_t lo = 0xffffffffu, hi = 0;
        for (uint64_t i = 0; i < n; ++i) {
                const uint32_t d = docids[i];
                if (d == 0)
                        return fail(c, TRN_ERR_ARG, "docID 0 is not a document");
                if (d > c->pc.max_docid)
                        continue; // as for the masked documents: a set may name documents this source does not hold
                words[d >> 5] |= 1u << (d & 31u);
                lo = std::min(lo, d);
                hi = std::max(hi, d);
        }
        DevBuf            bits;
        const cudaError_t e = bits.ensure(words.size() * 4);
        if (e != cudaSuccess) {
                (void)cudaGetLastError(); // an allocation failure is not sticky: clear it
                return fail(c, TRN_ERR_CAPACITY, std::string("trn_docset_create: ") + cudaGetErrorString(e));
        }
        CK(cudaMemcpyAsync(bits.p, words.data(), words.size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (slot == c->docsets.size())
                c->docsets.emplace_back();
        auto &D = c->docsets[slot];
        D.bits  = std::move(bits);
        D.lo    = lo;
        D.hi    = hi;
        D.live  = true;
        *handle = (c->docset_epoch & 0xffffu) << 16 | slot;
        return TRN_OK;
}

// the set behind a handle (TRN_OK), or why there is none
static int docset_of(trn_ctx *c, uint32_t h, const trn_ctx::DocSet *&out) {
        if ((h >> 16) != (c->docset_epoch & 0xffffu))
                return fail(c, TRN_ERR_STATE, "docID set " + std::to_string(h) + " belongs to an index this context no longer holds");
        const uint32_t slot = h & 0xffffu;
        if (slot >= c->docsets.size() || !c->docsets[slot].live)
                return fail(c, TRN_ERR_ARG, "docID set " + std::to_string(h) + " does not exist (destroyed?)");
        out = &c->docsets[slot];
        return TRN_OK;
}

extern "C" int trn_docset_destroy(trn_ctx *c, uint32_t handle) {
        if (!c)
                return TRN_ERR_ARG;
        const trn_ctx::DocSet *d = nullptr;
        if (const int rc = docset_of(c, handle, d); rc != TRN_OK)
                return rc;
        CK(cudaSetDevice(c->device));
        CK(cudaStreamSynchronize(c->stream)); // a batch in flight may still read it
        auto &D = c->docsets[handle & 0xffffu];
        D.bits.release();
        D.live = false;
        return TRN_OK;
}

// the device view of a batch's filters and each query's allow span.  false (nothing written): no query names a set
static int resolve_filters(trn_ctx *c, const trn_doc_filter *filters, uint32_t nq, std::vector<DevFilter> &dev, std::vector<uint2> &clip, bool &any) {
        any = false;
        if (!filters)
                return TRN_OK;
        for (uint32_t q = 0; q < nq && !any; ++q)
                any = filters[q].allow != TRN_DOCSET_NONE || filters[q].deny != TRN_DOCSET_NONE;
        if (!any)
                return TRN_OK;
        dev.assign(nq, DevFilter{nullptr, nullptr, 0u, 0xffffffffu});
        clip.assign(nq, uint2{0u, 0xffffffffu});
        for (uint32_t q = 0; q < nq; ++q) {
                const trn_ctx::DocSet *d = nullptr;
                if (filters[q].allow != TRN_DOCSET_NONE) {
                        if (const int rc = docset_of(c, filters[q].allow, d); rc != TRN_OK)
                                return fail(c, rc, "query " + std::to_string(q) + " allow: " + c->err);
                        dev[q].allow = d->bits.as<uint32_t>();
                        dev[q].lo = clip[q].x = d->lo;
                        dev[q].hi = clip[q].y = d->hi;
                }
                if (filters[q].deny != TRN_DOCSET_NONE) {
                        if (const int rc = docset_of(c, filters[q].deny, d); rc != TRN_OK)
                                return fail(c, rc, "query " + std::to_string(q) + " deny: " + c->err);
                        dev[q].deny = d->bits.as<uint32_t>();
                }
        }
        return TRN_OK;
}

extern "C" int trn_index_info_get(trn_ctx *c, trn_index_info *o) {
        if (!c || !o)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        o->codec           = c->pc.codec;
        o->nterms          = c->nterms;
        o->max_docid       = c->pc.max_docid;
        o->tile_docs       = 1u << c->pc.tile_shift;
        o->ntiles          = c->ntiles;
        o->block_docs      = c->block_docs;
        o->index_bytes     = c->index_bytes;
        o->directory_bytes = c->dir_bytes;
        o->total_blocks    = c->total_blocks;
        o->total_postings  = c->total_postings;
        o->dense_terms        = c->dense_terms;
        o->dense_bitmap_bytes = c->dense_bytes;
        o->probe_terms        = c->probe_terms;
        o->probe_bitmap_bytes = c->probe_bytes;
        return TRN_OK;
}

static DevIndex dev_index(trn_ctx *c) {
        DevIndex ix;
        ix.index      = c->d_index.as<uint8_t>();
        ix.blk_last   = c->d_blk_last.as<uint32_t>();
        ix.blk_off    = c->d_blk_off.as<uint32_t>();
        ix.terms      = c->d_terms.as<DevTerm>();
        ix.tile_first = c->d_tile_first.as<uint32_t>();
        ix.masked     = c->have_masked ? c->d_masked.as<uint32_t>() : nullptr;
        ix.nterms     = c->nterms;
        ix.ntiles     = c->ntiles;
        ix.tile_shift = c->pc.tile_shift;
        ix.max_docid  = c->pc.max_docid;
        ix.block_docs = c->block_docs;
        ix.codec      = c->pc.codec;
        ix.hits       = c->have_hits ? c->d_hits.as<uint8_t>() : nullptr;
        ix.hit_base   = c->have_hits ? c->d_hit_base.as<uint32_t>() : nullptr;
        ix.hblk_off   = c->have_hits ? c->d_hblk_off.as<uint32_t>() : nullptr;
        ix.hit_term   = c->have_hits ? c->d_hit_term.as<HitTerm>() : nullptr;
        const bool bitmaps = c->dense_terms || c->probe_terms;
        ix.dense      = bitmaps ? c->d_dense.as<uint32_t>() : nullptr;
        ix.dense_off  = c->dense_terms ? c->d_dense_off.as<uint32_t>() : nullptr;
        ix.probe_off  = bitmaps ? c->d_probe_off.as<uint32_t>() : nullptr;
        return ix;
}

// =================================================================================================== exec
// small device scratch layout (d_small): [0] ticket u32, [2..3] seg_cursor u64, [4] overflow u32, then per-query arrays.
// routes[0 .. nq): the TRN_ROUTE_* of every query (written on success)
// collect: non-null = the docs pass of the default exec mode (mode DOCS_ONLY; the plan is made in TRN_MODE_MATCHED_TERMS, and its collect
// programs are moved to *collect)
// filters: null, or one per query (trn_doc_filter)
static int exec_device_impl(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out, int set, cudaEvent_t k0, cudaEvent_t k1,
                            uint8_t *routes, const trn_doc_filter *filters, CollectPlan *collect = nullptr) {
        if (!c)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (!queries || !nq || mode < 0 || mode > 3)
                return fail(c, TRN_ERR_ARG, "trn_exec_batch: bad arguments");
        const bool compact = mode == TRN_MODE_DOCS_COMPACT; // DocumentsOnly with compact result segments; everything else is the same plan
        if (compact)
                mode = TRN_MODE_DOCS_ONLY;
        if (c->block_docs != (c->pc.codec == TRN_CODEC_GOOGLE ? 32u : 128u))
                return fail(c, TRN_ERR_UNSUPPORTED, "the uploaded index was built with a block size other than the reference format's (decode sweep only)");
        if (mode == TRN_MODE_SCORED_TOPK && (k == 0 || k > kernel_max_k()))
                return fail(c, TRN_ERR_ARG, "top-k: k must be in [1, 512]");
        CK(cudaSetDevice(c->device));
        const bool scored = mode != TRN_MODE_DOCS_ONLY;

        const double tCompile0 = now_ms();
        std::vector<DevFilter> devFilters;
        std::vector<uint2>     clip;
        bool                   filtered{false};
        if (const int rc = resolve_filters(c, filters, nq, devFilters, clip, filtered); rc != TRN_OK)
                return rc;
        c->pc.allow_phrase     = c->pc.codec == TRN_CODEC_GOOGLE || c->have_hits; // GOOGLE: inline hits; LUCENE: hits.data uploaded (trn_upload_hits)
        BatchPlan   plan;
        std::string perr;
        const int   prc = plan_batch(c->pc, c->h_terms, c->dense_terms ? c->h_dense_off.data() : nullptr, queries, nq, collect ? TRN_MODE_MATCHED_TERMS : mode, k, plan,
                                     perr, filtered ? clip.data() : nullptr, c->h_groups.base.empty() ? nullptr : &c->h_groups);
        if (prc != TRN_OK)
                return fail(c, prc, perr);
        if (collect)
                *collect = std::move(plan.collect);
        c->tm.host_compile_ms += float(now_ms() - tCompile0);
        const double   tEnqueue0  = now_ms();
        const uint32_t totalItems = uint32_t(plan.items);
        const uint32_t execShift  = plan.exec_shift;
        const uint64_t segCap     = plan.seg_cap;
        const auto &   steps      = plan.steps;

        // ---- result staging must fit the device: a caller (trn_exec_batch) reacts to TRN_ERR_CAPACITY by splitting the batch
        if (mode != TRN_MODE_SCORED_TOPK) {
                const uint64_t need = segCap * (scored ? 16ull : 8ull) + uint64_t(totalItems) * 20ull;
                const uint64_t have = c->d_seg_docids.cap + c->d_out_docids[set].cap + c->d_seg_scores.cap + c->d_out_scores[set].cap;
                if (need > have) {
                        size_t freeB{0}, totalB{0};
                        CK(cudaMemGetInfo(&freeB, &totalB));
                        if (need - have > uint64_t(double(freeB) * 0.8))
                                return fail(c, TRN_ERR_CAPACITY, "batch needs " + std::to_string(need >> 20) + " MiB of result staging (upper bound of the matches); split it");
                }
        }

        // ---- device buffers
        CK(c->d_queries.ensure(nq * sizeof(DevQuery)));
        CK(c->d_steps.ensure(std::max<size_t>(sizeof(DevStep), steps.size() * sizeof(DevStep))));
        const size_t smallBytes = 64 + size_t(nq) * (8 + 4 + 4 + 8);
        CK(c->d_small[set].ensure(smallBytes));
        CK(c->d_q_offsets[set].ensure((size_t(nq) + 1) * 8));
        if (mode != TRN_MODE_SCORED_TOPK) {
                CK(c->d_item_off.ensure(std::max<size_t>(8, size_t(totalItems) * 8)));
                CK(c->d_item_cnt.ensure(std::max<size_t>(4, size_t(totalItems) * 4)));
                CK(c->d_item_dst.ensure(std::max<size_t>(8, size_t(totalItems) * 8)));
                CK(c->d_seg_docids.ensure(std::max<size_t>(4, segCap * 4)));
                CK(c->d_out_docids[set].ensure(std::max<size_t>(4, segCap * 4)));
                if (scored) {
                        CK(c->d_seg_scores.ensure(std::max<size_t>(4, segCap * 4)));
                        CK(c->d_out_scores[set].ensure(std::max<size_t>(4, segCap * 4)));
                }
        } else {
                CK(c->d_cand.ensure(std::max<size_t>(8, plan.cand_total * 8)));
                CK(c->d_topk_docids.ensure(size_t(nq) * k * 4));
                CK(c->d_topk_scores.ensure(size_t(nq) * k * 4));
                CK(c->d_topk_counts.ensure(size_t(nq) * 4));
        }
        const uint32_t nflat = uint32_t(plan.flat.size());
        if (nflat) {
                CK(c->d_fq.ensure(plan.flat.size() * sizeof(FlatQuery)));
                CK(c->d_leaves.ensure(plan.leaves.size() * sizeof(FlatLeaf)));
                CK(c->d_luts.ensure(plan.leaves.size() * 64 * sizeof(float)));
                CK(cudaMemcpyAsync(c->d_fq.p, plan.flat.data(), plan.flat.size() * sizeof(FlatQuery), cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(c->d_leaves.p, plan.leaves.data(), plan.leaves.size() * sizeof(FlatLeaf), cudaMemcpyHostToDevice, c->stream));
        }
        uint8_t *small        = c->d_small[set].as<uint8_t>();
        auto *   ticket       = reinterpret_cast<uint32_t *>(small);
        auto *   seg_cursor   = reinterpret_cast<unsigned long long *>(small + 8);
        auto *   overflow     = reinterpret_cast<uint32_t *>(small + 16);
        auto *   match_counts = reinterpret_cast<unsigned long long *>(small + 64);
        auto *   theta        = reinterpret_cast<uint32_t *>(small + 64 + size_t(nq) * 8);
        auto *   cand_cursor  = reinterpret_cast<uint32_t *>(small + 64 + size_t(nq) * 12);
        auto *   word_counts  = reinterpret_cast<unsigned long long *>(small + 64 + size_t(nq) * 16);

        if (set < 0 || set > 1)
                return TRN_ERR_ARG;
        if (compact) {
                CK(c->d_item_desc[set].ensure(std::max<size_t>(4, size_t(totalItems) * 4)));
                auto &qi = c->qitems_set[set];
                qi.resize(nq);
                for (uint32_t q = 0; q < nq; ++q) {
                        const DevQuery &dq = plan.queries[q];
                        qi[q] = trn_qitems{dq.item_base, dq.ntiles, dq.tile_lo, dq.route == TRN_ROUTE_FLAT_TREE ? c->pc.tree_shift : execShift};
                }
        }
        CK(cudaMemcpyAsync(c->d_queries.p, plan.queries.data(), nq * sizeof(DevQuery), cudaMemcpyHostToDevice, c->stream));
        if (filtered) {
                CK(c->d_filters.ensure(nq * sizeof(DevFilter)));
                CK(cudaMemcpyAsync(c->d_filters.p, devFilters.data(), nq * sizeof(DevFilter), cudaMemcpyHostToDevice, c->stream));
        }
        if (!steps.empty())
                CK(cudaMemcpyAsync(c->d_steps.p, steps.data(), steps.size() * sizeof(DevStep), cudaMemcpyHostToDevice, c->stream));
        const uint32_t denseItems = uint32_t(plan.dense_runs.size());
        if (denseItems) {
                CK(c->d_dense_runs.ensure(size_t(denseItems) * sizeof(uint2)));
                CK(cudaMemcpyAsync(c->d_dense_runs.p, plan.dense_runs.data(), size_t(denseItems) * sizeof(uint2), cudaMemcpyHostToDevice, c->stream));
        }
        const uint32_t mixedItems = uint32_t(plan.mixed_runs.size());
        if (mixedItems) {
                CK(c->d_mixed_runs.ensure(size_t(mixedItems) * sizeof(uint2)));
                CK(cudaMemcpyAsync(c->d_mixed_runs.p, plan.mixed_runs.data(), size_t(mixedItems) * sizeof(uint2), cudaMemcpyHostToDevice, c->stream));
        }
        const uint32_t candItems = uint32_t(plan.cand_order.size());
        if (candItems) {
                CK(c->d_cand_order.ensure(size_t(candItems) * sizeof(uint32_t)));
                CK(cudaMemcpyAsync(c->d_cand_order.p, plan.cand_order.data(), size_t(candItems) * sizeof(uint32_t), cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaMemsetAsync(small, 0, smallBytes, c->stream));

        ExecParams P;
        std::memset(&P, 0, sizeof(P));
        P.ix           = dev_index(c);
        P.queries      = c->d_queries.as<DevQuery>();
        P.steps        = c->d_steps.as<DevStep>();
        P.nq           = nq;
        P.total_items  = totalItems;
        P.gen_items    = uint32_t(plan.gen_items);
        P.dense_runs   = denseItems ? c->d_dense_runs.as<uint2>() : nullptr;
        P.dense_items  = denseItems;
        P.mixed_runs   = mixedItems ? c->d_mixed_runs.as<uint2>() : nullptr;
        P.mixed_items  = mixedItems;
        P.cand_order   = candItems ? c->d_cand_order.as<uint32_t>() : nullptr;
        P.cand_items   = candItems;
        P.has_phrase   = plan.any_phrase ? 1u : 0u;
        P.nslots       = plan.nslots;
        P.exec_shift   = execShift;
        P.stage_bytes  = exec_stage_bytes(c->pc.codec);
        P.docs_stage_bytes = exec_docs_stage_bytes();
        P.mode         = mode;
        P.k            = k;
        P.ticket       = ticket;
        P.seg_cursor   = seg_cursor;
        P.seg_capacity = segCap;
        P.seg_docids   = c->d_seg_docids.as<uint32_t>();
        P.seg_scores   = scored ? c->d_seg_scores.as<float>() : nullptr;
        P.item_off     = c->d_item_off.as<uint64_t>();
        P.item_cnt     = c->d_item_cnt.as<uint32_t>();
        P.item_desc    = compact ? c->d_item_desc[set].as<uint32_t>() : nullptr;
        P.word_counts  = word_counts;
        P.match_counts = match_counts;
        P.theta        = theta;
        P.cand_cursor  = cand_cursor;
        P.cand         = c->d_cand.as<uint2>();
        P.overflow     = overflow;
        P.filters      = filtered ? c->d_filters.as<DevFilter>() : nullptr;

        uint32_t launches{0};
        if (totalItems) {
                const bool     warpKernel = !scored;
                const uint64_t ownItems   = plan.gen_items + denseItems + mixedItems + candItems; // tickets of the step-program launch
                CK(cudaEventRecord(k0, c->stream));
                if (nflat && plan.flat_items) {
                        // flat scored disjunctions: per-leaf BM25 tables once per batch, then k_score_flat
                        ScoreParams S;
                        std::memset(&S, 0, sizeof(S));
                        S.ix           = P.ix;
                        S.fq           = c->d_fq.as<FlatQuery>();
                        S.leaves       = c->d_leaves.as<FlatLeaf>();
                        S.luts         = c->d_luts.as<float>();
                        S.nflat        = nflat;
                        S.run_tiles    = c->pc.run_tiles;
                        S.total_items  = mode == TRN_MODE_SCORED_TOPK ? uint32_t(std::min<uint64_t>(uint64_t(plan.max_runs) * nflat, 0xffffffffull)) : uint32_t(plan.flat_items);
                        S.tile_shift   = c->pc.scored_shift;
                        S.mode         = mode;
                        S.k            = k;
                        S.ticket       = reinterpret_cast<uint32_t *>(small + 4);
                        S.match_counts = match_counts;
                        S.theta        = theta;
                        S.cand_cursor  = cand_cursor;
                        S.cand         = P.cand;
                        S.seg_cursor   = seg_cursor;
                        S.seg_capacity = segCap;
                        S.seg_docids   = P.seg_docids;
                        S.seg_scores   = P.seg_scores;
                        S.item_off     = P.item_off;
                        S.item_cnt     = P.item_cnt;
                        S.overflow     = overflow;
                        S.filters      = P.filters;
                        CK(launch_build_luts(S.leaves, uint32_t(plan.leaves.size()), c->d_luts.as<float>(), c->stream));
                        CK(launch_score_flat(S, c->flat_threads, c->num_sms, c->stream));
                        launches += 2;
                }
                if (ownItems) {
                        const int perSM = warpKernel ? exec_docs_max_ctas_per_sm(execShift, plan.nslots, exec_docs_stage_bytes(), false, c->pc.codec == TRN_CODEC_LUCENE, filtered)
                                                     : exec_max_ctas_per_sm(execShift, plan.nslots, mode, c->pc.codec, filtered);
                        if (perSM <= 0)
                                return fail(c, TRN_ERR_CUDA, "the exec kernel does not fit on an SM with this many docset slots");
                        const uint64_t workers = warpKernel ? (ownItems + 3) / 4 : ownItems; // 4 warp-workers per CTA
                        const int      grid    = int(std::min<uint64_t>(uint64_t(c->num_sms) * perSM, std::max<uint64_t>(1, workers)));
                        if (warpKernel)
                                CK(launch_exec_docs(P, grid, c->stream));
                        else
                                CK(launch_exec_tiles(P, grid, c->stream));
                        ++launches;
                }
                if (warpKernel && plan.gen_items2) { // flat-tree plans: same kernel, own tile size / slot count / ticket space
                        ExecParams P2 = P;
                        P2.exec_shift = c->pc.tree_shift;
                        P2.nslots     = plan.tree_slots;
                        P2.gen_items  = uint32_t(plan.gen_items2);
                        P2.gen_sel    = 1;
                        P2.dense_runs  = nullptr;
                        P2.dense_items = 0;
                        P2.mixed_runs  = nullptr;
                        P2.mixed_items = 0;
                        P2.cand_order  = nullptr;
                        P2.cand_items  = 0;
                        P2.ticket     = reinterpret_cast<uint32_t *>(small + 4);
                        const int perSM = exec_docs_max_ctas_per_sm(P2.exec_shift, P2.nslots, exec_docs_stage_bytes(), true, false, filtered);
                        if (perSM <= 0)
                                return fail(c, TRN_ERR_CUDA, "the flat-tree launch does not fit on an SM with this many docset slots");
                        const int grid = int(std::min<uint64_t>(uint64_t(c->num_sms) * perSM, std::max<uint64_t>(1, (plan.gen_items2 + 3) / 4)));
                        CK(launch_exec_docs(P2, grid, c->stream));
                        ++launches;
                }
                CK(cudaEventRecord(k1, c->stream));
                c->have_kernel_events = true;
        } else {
                CK(cudaEventRecord(k0, c->stream)); // keep the pair fresh: readers must not see a previous batch's events
                CK(cudaEventRecord(k1, c->stream));
        }
        if (mode != TRN_MODE_SCORED_TOPK) {
                CK(launch_query_scan(compact ? word_counts : match_counts, nq, c->d_q_offsets[set].as<uint64_t>(), c->stream)); // compact: offsets in words
                ++launches;
                if (totalItems) {
                        CK(launch_item_scan(P.queries, nq, P.item_cnt, c->d_q_offsets[set].as<uint64_t>(), c->d_item_dst.as<uint64_t>(), c->stream));
                        CK(launch_gather(totalItems, P.item_off, P.item_cnt, c->d_item_dst.as<uint64_t>(), P.seg_docids, P.seg_scores,
                                         c->d_out_docids[set].as<uint32_t>(), scored ? c->d_out_scores[set].as<float>() : nullptr, c->stream));
                        launches += 2;
                }
        } else {
                CK(launch_topk_select(P.queries, nq, P.cand, cand_cursor, k, c->d_topk_docids.as<uint32_t>(), c->d_topk_scores.as<float>(),
                                      c->d_topk_counts.as<uint32_t>(), c->stream));
                ++launches;
        }
        c->tm.enqueue_ms += float(now_ms() - tEnqueue0);
        c->last_mode     = compact ? TRN_MODE_DOCS_COMPACT : mode;
        c->last_items    = totalItems;
        c->last_nq       = nq;
        c->last_k        = k;
        c->last_launches = launches;
        c->last_postings = plan.postings;
        c->last_bytes    = plan.bytes;
        if (out) {
                std::memset(out, 0, sizeof(*out));
                out->nq                  = nq;
                out->postings_scanned    = plan.postings;
                out->index_bytes_touched = plan.bytes;
                out->kernel_launches     = launches;
        }
        for (uint32_t q = 0; q < nq; ++q)
                routes[q] = uint8_t(plan.queries[q].route);
        return TRN_OK;
}

extern "C" int trn_exec_batch_device(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out) {
        return trn_exec_batch_device_filtered(c, queries, nq, mode, k, nullptr, out);
}

extern "C" int trn_exec_batch_device_filtered(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, const trn_doc_filter *filters, trn_result *out) {
        if (!c)
                return TRN_ERR_ARG;
        CK(cudaSetDevice(c->device));
        c->have_kernel_events = false;
        c->tm                 = trn_timings{};
        c->last_routes.clear();
        const double t0       = now_ms();
        CK(cudaEventRecord(c->ev0, c->stream));
        std::vector<uint8_t> routes(nq);
        const int            r = exec_device_impl(c, queries, nq, mode, k, out, 0, c->evk0, c->evk1, routes.data(), filters);
        c->tm.total_ms = float(now_ms() - t0);
        if (r != TRN_OK)
                return r;
        c->last_routes = std::move(routes);
        CK(cudaEventRecord(c->ev1, c->stream));
        return TRN_OK;
}

extern "C" int trn_fetch_results(trn_ctx *c, trn_result *out) {
        if (!c || !out)
                return TRN_ERR_ARG;
        if (c->last_mode < 0)
                return fail(c, TRN_ERR_STATE, "no batch executed");
        CK(cudaSetDevice(c->device));
        const uint32_t nq = c->last_nq;
        const uint8_t *small        = c->d_small[0].as<uint8_t>();
        const auto *   match_counts = reinterpret_cast<const unsigned long long *>(small + 64);
        CK(c->h_offsets.ensure((size_t(nq) + 1) * 8));
        CK(c->h_counts.ensure(size_t(nq) * 8));
        CK(c->h_small.ensure(64 + size_t(nq) * 4));
        CK(cudaMemcpyAsync(c->h_counts.p, match_counts, size_t(nq) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(c->h_small.p, small, 64, cudaMemcpyDeviceToHost, c->stream));
        std::memset(out, 0, sizeof(*out));
        out->nq = nq;
        if (c->last_mode != TRN_MODE_SCORED_TOPK) {
                CK(cudaMemcpyAsync(c->h_offsets.p, c->d_q_offsets[0].p, (size_t(nq) + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                if (c->h_small.as<uint32_t>()[4])
                        return fail(c, TRN_ERR_CAPACITY, "segment buffer overflow (internal bound violated)");
                const uint64_t total = c->h_offsets.as<uint64_t>()[nq];
                CK(c->h_docids.ensure(std::max<size_t>(4, total * 4)));
                if (total)
                        CK(cudaMemcpyAsync(c->h_docids.p, c->d_out_docids[0].p, total * 4, cudaMemcpyDeviceToHost, c->stream));
                if (c->last_mode == TRN_MODE_SCORED_ALL) {
                        CK(c->h_scores.ensure(std::max<size_t>(4, total * 4)));
                        if (total)
                                CK(cudaMemcpyAsync(c->h_scores.p, c->d_out_scores[0].p, total * 4, cudaMemcpyDeviceToHost, c->stream));
                        out->scores = c->h_scores.as<float>();
                }
                if (c->last_mode == TRN_MODE_DOCS_COMPACT) {
                        CK(c->h_item_desc.ensure(std::max<size_t>(4, size_t(c->last_items) * 4)));
                        if (c->last_items)
                                CK(cudaMemcpyAsync(c->h_item_desc.p, c->d_item_desc[0].p, size_t(c->last_items) * 4, cudaMemcpyDeviceToHost, c->stream));
                }
                CK(cudaStreamSynchronize(c->stream));
                if (c->last_mode == TRN_MODE_DOCS_COMPACT) {
                        c->h_qitems      = c->qitems_set[0];
                        out->words       = c->h_docids.as<uint32_t>();
                        out->total_words = total;
                        out->item_desc   = c->h_item_desc.as<uint32_t>();
                        out->qitems      = c->h_qitems.data();
                        uint64_t matches{0};
                        for (uint32_t q = 0; q < nq; ++q)
                                matches += c->h_counts.as<uint64_t>()[q];
                        out->total = matches;
                } else {
                        out->total  = total;
                        out->docids = c->h_docids.as<uint32_t>();
                }
        } else {
                const uint32_t k = c->last_k;
                CK(c->h_docids.ensure(size_t(nq) * k * 4));
                CK(c->h_scores.ensure(size_t(nq) * k * 4));
                uint32_t *hc = c->h_small.as<uint32_t>() + 16;
                CK(cudaMemcpyAsync(c->h_docids.p, c->d_topk_docids.p, size_t(nq) * k * 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(c->h_scores.p, c->d_topk_scores.p, size_t(nq) * k * 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(hc, c->d_topk_counts.p, size_t(nq) * 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                // fixed stride k per query: offsets[q] = q*k, valid entries = counts
                uint64_t *off = c->h_offsets.as<uint64_t>();
                uint64_t  tot{0};
                for (uint32_t q = 0; q < nq; ++q) {
                        off[q] = uint64_t(q) * k;
                        tot += hc[q];
                }
                off[nq]     = uint64_t(nq) * k;
                out->total  = tot;
                out->docids = c->h_docids.as<uint32_t>();
                out->scores = c->h_scores.as<float>();
        }
        out->offsets             = c->h_offsets.as<uint64_t>();
        out->match_counts        = c->h_counts.as<uint64_t>();
        out->postings_scanned    = c->last_postings;
        out->index_bytes_touched = c->last_bytes;
        out->kernel_launches     = c->last_launches;
        float ms{0};
        if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) == cudaSuccess)
                out->device_ms = ms;
        if (c->have_kernel_events && cudaEventElapsedTime(&ms, c->evk0, c->evk1) == cudaSuccess)
                out->exec_kernel_ms = ms;
        return TRN_OK;
}

// Host-buffer entry point.  DOCS_ONLY / SCORED_ALL batches are split into chunks: the fused kernels of chunk i+1 run while the
// results of chunk i travel to the (pinned) host buffer on a second stream — the e2e time tends to max(kernels, D2H) instead of
// their sum.  Output-side device buffers are double-buffered (set = chunk parity); everything else is reused in stream order.
extern "C" int trn_exec_batch(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out) {
        return trn_exec_batch_filtered(c, queries, nq, mode, k, nullptr, out);
}

extern "C" int trn_exec_batch_filtered(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, const trn_doc_filter *filters, trn_result *out) {
        if (!c || !out)
                return TRN_ERR_ARG;
        if (filters) { // every handle is checked before the first chunk is launched
                std::vector<DevFilter> dev;
                std::vector<uint2>     clip;
                bool                   any{false};
                if (const int rc = resolve_filters(c, filters, nq, dev, clip, any); rc != TRN_OK)
                        return rc;
        }
        // how the batch is split into pipelined launches: chunkplan.h (a pure function of what is known here, pinned on the CPU by
        // tests/test_chunk_plan_cpu.py).
        ChunkPlanIn pin;
        pin.nq   = nq;
        pin.topk = mode == TRN_MODE_SCORED_TOPK;
        if (queries && c->have_index)
                for (uint32_t q = 0; q < nq; ++q)
                        for (uint32_t i = 0; i < queries[q].nnodes && queries[q].nodes; ++i)
                                if (queries[q].nodes[i].kind == TRN_NODE_TERM && queries[q].nodes[i].term < c->nterms) {
                                        pin.est_postings += c->h_terms[queries[q].nodes[i].term].documents;
                                        ++pin.leaves;
                                }
        pin.max_chunks      = (queries && c->have_index) ? c->pipeline_chunks : 1u;
        pin.chunk_postings  = c->chunk_postings;
        pin.rule_sqrt       = c->chunk_rule_sqrt;
        pin.taper           = c->taper_chunks;
        pin.tail_ms         = c->chunk_tail_ms;
        pin.tail_tree_ms    = c->chunk_tail_tree_ms;
        pin.hint_bytes      = c->hint_bytes;
        pin.hint_postings   = c->hint_postings;
        pin.hint_same_shape = c->hint_nq == nq && c->hint_mode == mode;
        const ChunkPlan plan        = plan_chunks(pin);
        const uint64_t  estPostings = pin.est_postings;
        const bool      compact     = mode == TRN_MODE_DOCS_COMPACT;
        if (plan.single_call) {
                const double t0 = now_ms();
                const int    r  = trn_exec_batch_device_filtered(c, queries, nq, mode, k, filters, nullptr);
                if (r != TRN_OK)
                        return r;
                const double tw = now_ms();
                const int    fr = trn_fetch_results(c, out);
                c->tm.final_wait_ms = float(now_ms() - tw);
                c->tm.total_ms      = float(now_ms() - t0);
                c->tm.chunks        = 1.f;
                if (fr == TRN_OK && mode != TRN_MODE_SCORED_TOPK) { // (a batch that took the single-call form still tells the next one its size)
                        c->hint_bytes    = (compact ? out->total_words : out->total) * 4 * (mode == TRN_MODE_SCORED_ALL ? 2 : 1);
                        c->hint_nq       = nq;
                        c->hint_mode     = mode;
                        c->hint_postings = estPostings;
                }
                if (fr == TRN_OK)
                        c->tm.kernel_ms = out->exec_kernel_ms;
                return fr;
        }
        CK(cudaSetDevice(c->device));
        c->tm            = trn_timings{};
        c->last_routes.clear();
        std::vector<uint8_t> routes(nq, 0);
        const double tB0 = now_ms();
        const bool scored = mode == TRN_MODE_SCORED_ALL;
        CK(c->h_offsets.ensure((size_t(nq) + 1) * 8));
        CK(c->h_counts.ensure(size_t(nq) * 8));
        const uint32_t per = *std::max_element(plan.sizes.begin(), plan.sizes.end()); // queries of the largest launch
        CK(c->h_chunk.ensure(2 * (64 + (size_t(per) + 1) * 16)));
        uint64_t *hoff = c->h_offsets.as<uint64_t>(), *hcnt = c->h_counts.as<uint64_t>();
        uint64_t  running{0}, postings{0}, bytes{0}, runningItems{0}, matches{0};
        uint32_t  launches{0};
        std::vector<uint32_t> chunkItems; // compact: work items of every chunk (entries of its item_desc)
        if (compact)
                c->h_qitems.resize(nq);
        float     ksum{0};
        struct Chunk {
                uint32_t q0, n;
        };
        std::vector<Chunk> ch;
        {
                uint32_t q0{0};
                for (const uint32_t n : plan.sizes) {
                        ch.push_back({q0, n});
                        q0 += n;
                }
        }
        auto finish = [&](uint32_t j) -> int {
                const int   set = int(j & 1);
                const auto &C   = ch[j];
                uint8_t *   hs  = c->h_chunk.as<uint8_t>() + size_t(set) * (64 + (size_t(per) + 1) * 16);
                uint64_t *  o   = reinterpret_cast<uint64_t *>(hs + 64);
                uint64_t *  m   = o + per + 1;
                const uint8_t *small = c->d_small[set].as<uint8_t>();
                CK(cudaStreamWaitEvent(c->copy_stream, c->ev_done[set], 0));
                CK(cudaMemcpyAsync(hs, small, 64, cudaMemcpyDeviceToHost, c->copy_stream));
                CK(cudaMemcpyAsync(o, c->d_q_offsets[set].p, (size_t(C.n) + 1) * 8, cudaMemcpyDeviceToHost, c->copy_stream));
                CK(cudaMemcpyAsync(m, small + 64, size_t(C.n) * 8, cudaMemcpyDeviceToHost, c->copy_stream));
                {
                        const double tw = now_ms(); // waits for the chunk's kernels (and the previous chunk's result copy on the same stream)
                        CK(cudaStreamSynchronize(c->copy_stream));
                        c->tm.chunk_wait_ms += float(now_ms() - tw);
                }
                {
                        float kms{0}; // the chunk's kernels are complete: its event pair can be read (and its slot reused 16 chunks later)
                        if (cudaEventElapsedTime(&kms, c->ev_ck0[j % 16], c->ev_ck1[j % 16]) == cudaSuccess)
                                ksum += kms;
                }
                if (reinterpret_cast<uint32_t *>(hs)[4])
                        return fail(c, TRN_ERR_CAPACITY, "segment buffer overflow (internal bound violated)");
                const uint64_t total = o[C.n];
                // grow-only pinned result buffers; after the first batch the previous total is the hint that avoids regrowth
                const size_t need = std::max<size_t>(4, std::max<uint64_t>(running + total, c->last_total_hint) * 4);
                CK(c->h_docids.grow(need, running * 4, c->copy_stream));
                if (scored)
                        CK(c->h_scores.grow(need, running * 4, c->copy_stream));
                if (total) {
                        CK(cudaMemcpyAsync(c->h_docids.as<uint32_t>() + running, c->d_out_docids[set].p, total * 4, cudaMemcpyDeviceToHost, c->copy_stream));
                        if (scored)
                                CK(cudaMemcpyAsync(c->h_scores.as<float>() + running, c->d_out_scores[set].p, total * 4, cudaMemcpyDeviceToHost, c->copy_stream));
                }
                if (compact) { // the chunk's segment descriptors; its queries' item ranges move behind the earlier chunks' items
                        const uint32_t ni = chunkItems[j];
                        CK(c->h_item_desc.grow(std::max<size_t>(4, std::max<uint64_t>(runningItems + ni, c->last_items_hint) * 4), runningItems * 4, c->copy_stream));
                        if (ni)
                                CK(cudaMemcpyAsync(c->h_item_desc.as<uint32_t>() + runningItems, c->d_item_desc[set].p, size_t(ni) * 4, cudaMemcpyDeviceToHost, c->copy_stream));
                        for (uint32_t i = 0; i < C.n; ++i) {
                                trn_qitems qi = c->qitems_chunk[j][i];
                                qi.item_base += uint32_t(runningItems);
                                c->h_qitems[C.q0 + i] = qi;
                        }
                        runningItems += ni;
                }
                CK(cudaEventRecord(c->ev_d2h[set], c->copy_stream));
                for (uint32_t i = 0; i < C.n; ++i) {
                        hoff[C.q0 + i] = running + o[i];
                        hcnt[C.q0 + i] = m[i];
                        matches += m[i];
                }
                running += total;
                return TRN_OK;
        };
        CK(cudaEventRecord(c->ev0, c->stream));
        for (uint32_t i = 0; i < ch.size(); ++i) {
                const int set = int(i & 1);
                if (i >= 2)
                        CK(cudaStreamWaitEvent(c->stream, c->ev_d2h[set], 0)); // the set's previous results have left the device
                trn_result part;
                const int  r = exec_device_impl(c, queries + ch[i].q0, ch[i].n, mode, k, &part, set, c->ev_ck0[i % 16], c->ev_ck1[i % 16], routes.data() + ch[i].q0,
                                                filters ? filters + ch[i].q0 : nullptr);
                if (r == TRN_ERR_CAPACITY && ch[i].n > 1) {
                        // the upper bound of this chunk's matches does not fit the device: halve it and retry (nothing was launched)
                        const Chunk a{ch[i].q0, ch[i].n / 2}, b{ch[i].q0 + ch[i].n / 2, ch[i].n - ch[i].n / 2};
                        ch[i] = a;
                        ch.insert(ch.begin() + i + 1, b);
                        --i;
                        continue;
                }
                if (r != TRN_OK)
                        return r;
                CK(cudaEventRecord(c->ev_done[set], c->stream));
                if (compact) {
                        if (chunkItems.size() <= i) {
                                chunkItems.resize(i + 1);
                                c->qitems_chunk.resize(i + 1);
                        }
                        chunkItems[i]      = c->last_items;
                        c->qitems_chunk[i] = c->qitems_set[set];
                }
                postings += part.postings_scanned;
                bytes += part.index_bytes_touched;
                launches += part.kernel_launches;
                if (i >= 1) {
                        const int fr = finish(i - 1);
                        if (fr != TRN_OK)
                                return fr;
                }
        }
        CK(cudaEventRecord(c->ev1, c->stream));
        {
                const int fr = finish(uint32_t(ch.size()) - 1);
                if (fr != TRN_OK)
                        return fr;
        }
        {
                const double tw = now_ms();
                CK(cudaStreamSynchronize(c->copy_stream));
                CK(cudaStreamSynchronize(c->stream));
                c->tm.final_wait_ms = float(now_ms() - tw);
        }
        c->tm.total_ms     = float(now_ms() - tB0);
        c->tm.kernel_ms    = ksum;
        c->tm.chunks       = float(ch.size());
        hoff[nq]           = running;
        c->last_total_hint = running + running / 16;
        c->hint_bytes      = running * 4 * (scored ? 2 : 1);
        c->hint_nq         = nq;
        c->hint_mode       = mode;
        c->hint_postings   = estPostings;
        std::memset(out, 0, sizeof(*out));
        out->nq                  = nq;
        out->total               = compact ? matches : running;
        out->offsets             = hoff;
        out->docids              = compact ? nullptr : c->h_docids.as<uint32_t>();
        out->scores              = scored ? c->h_scores.as<float>() : nullptr;
        if (compact) {
                out->words         = c->h_docids.as<uint32_t>();
                out->total_words   = running;
                out->item_desc     = c->h_item_desc.as<uint32_t>();
                out->qitems        = c->h_qitems.data();
                c->last_items_hint = runningItems + runningItems / 16;
        }
        out->match_counts        = hcnt;
        out->postings_scanned    = postings;
        out->index_bytes_touched = bytes;
        out->kernel_launches     = launches;
        float ms{0};
        if (cudaEventElapsedTime(&ms, c->ev0, c->ev1) == cudaSuccess)
                out->device_ms = ms;
        out->exec_kernel_ms = ksum;
        // the split-form API (trn_fetch_results / trn_last_topk_device) refers to a whole batch; a pipelined call leaves none behind
        c->last_mode   = -1;
        c->last_routes = std::move(routes);
        return TRN_OK;
}

extern "C" int trn_debug_last_routes(trn_ctx *c, uint8_t *out, uint32_t cap, uint32_t *n) {
        if (!c || !n)
                return TRN_ERR_ARG;
        *n = uint32_t(c->last_routes.size());
        if (cap < *n)
                return fail(c, TRN_ERR_CAPACITY, "trn_debug_last_routes: buffer too small");
        if (*n)
                std::memcpy(out, c->last_routes.data(), *n);
        return TRN_OK;
}

// plans a batch on the host as exec_device_impl would on a context that holds this index (trn_debug_plan, trn_debug_dense_runs)
// ============================================================================================ default exec mode
extern "C" int trn_exec_matches(trn_ctx *c, const trn_query *queries, uint32_t nq, trn_matches *out) {
        return trn_exec_matches_filtered(c, queries, nq, nullptr, out);
}

extern "C" int trn_exec_matches_filtered(trn_ctx *c, const trn_query *queries, uint32_t nq, const trn_doc_filter *filters, trn_matches *out) {
        if (!c || !out)
                return TRN_ERR_ARG;
        CK(cudaSetDevice(c->device));
        std::memset(out, 0, sizeof(*out));
        c->have_kernel_events = false;
        c->tm                 = trn_timings{};
        c->last_routes.clear();
        c->last_mode = -1;
        auto &M      = c->mt;
        if (!M.ev_docs) {
                for (Event *e : {&M.ev_docs, &M.ev_c0, &M.ev_c1, &M.ev_w0, &M.ev_w1, &M.ev_end})
                        CK(cudaEventCreate(&e->h));
        }
        const double t0 = now_ms();
        // ---- docs pass: the DocumentsOnly routes (root-filter quirk off) into d_out_docids[0] / d_q_offsets[0]
        CK(cudaEventRecord(c->ev0, c->stream));
        std::vector<uint8_t> routes(nq);
        CollectPlan          cp;
        const int            r = exec_device_impl(c, queries, nq, TRN_MODE_DOCS_ONLY, 0, nullptr, 0, c->evk0, c->evk1, routes.data(), filters, &cp);
        c->last_mode         = -1; // trn_fetch_results has nothing to fetch after this call (the docs pass leaves no trn_result)
        if (r != TRN_OK)
                return r;
        CK(cudaEventRecord(M.ev_docs, c->stream));
        CK(M.h_doc_off.ensure((size_t(nq) + 1) * 8));
        CK(cudaMemcpyAsync(M.h_doc_off.p, c->d_q_offsets[0].p, (size_t(nq) + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(M.h_small.ensure(64));
        CK(cudaMemcpyAsync(M.h_small.p, c->d_small[0].p, 64, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (M.h_small.as<uint32_t>()[4])
                return fail(c, TRN_ERR_CAPACITY, "segment buffer overflow (internal bound violated)");
        const uint64_t nm = M.h_doc_off.as<uint64_t>()[nq];
        CK(M.h_docids.ensure(std::max<size_t>(4, nm * 4)));
        if (nm)
                CK(cudaMemcpyAsync(M.h_docids.p, c->d_out_docids[0].p, nm * 4, cudaMemcpyDeviceToHost, c->stream));

        // ---- collect programs; per match of the batch: mask, term and hit counts and their scans (28 bytes)
        auto upload = [&](DevBuf &b, const void *src, size_t bytes) -> cudaError_t {
                if (const cudaError_t e = b.ensure(std::max<size_t>(16, bytes)); e != cudaSuccess)
                        return e;
                return bytes ? cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, c->stream) : cudaSuccess;
        };
        CK(upload(M.d_cq, cp.queries.data(), cp.queries.size() * sizeof(CollectQuery)));
        CK(upload(M.d_cterms, cp.terms.data(), cp.terms.size() * 4));
        CK(upload(M.d_cphrases, cp.phrases.data(), cp.phrases.size() * sizeof(CollectPhrase)));
        CK(upload(M.d_cargs, cp.args.data(), cp.args.size() * sizeof(DevStep)));
        CK(upload(M.d_cprog, cp.prog.data(), cp.prog.size() * sizeof(CollectOp)));
        CK(M.d_error.ensure(4));
        CK(cudaMemsetAsync(M.d_error.p, 0, 4, c->stream));
        for (DevBuf *b : {&M.d_mask, &M.d_nterms, &M.d_nhits})
                CK(b->ensure(std::max<size_t>(4, nm * 4)));
        for (DevBuf *b : {&M.d_tscan, &M.d_hscan})
                CK(b->ensure((nm + 1) * 8));
        CK(M.d_part.ensure((nm / 4096 + 2) * 8));

        CollectParams P;
        std::memset(&P, 0, sizeof(P));
        P.ix        = dev_index(c);
        P.queries   = M.d_cq.as<CollectQuery>();
        P.terms     = M.d_cterms.as<uint32_t>();
        P.phrases   = M.d_cphrases.as<CollectPhrase>();
        P.args      = M.d_cargs.as<DevStep>();
        P.prog      = M.d_cprog.as<CollectOp>();
        P.q_offsets = c->d_q_offsets[0].as<uint64_t>();
        P.docids    = c->d_out_docids[0].as<uint32_t>();
        P.nq        = nq;
        P.error     = M.d_error.as<uint32_t>();
        P.mask      = M.d_mask.as<uint32_t>();
        P.nterms    = M.d_nterms.as<uint32_t>();
        P.nhits     = M.d_nhits.as<uint32_t>();
        P.term_scan = M.d_tscan.as<unsigned long long>();
        P.hit_scan  = M.d_hscan.as<unsigned long long>();
        P.m0        = 0;
        P.m1        = nm;
        CK(cudaEventRecord(M.ev_c0, c->stream));
        CK(launch_collect_count(P, c->stream));
        CK(launch_enc_scan(P.nterms, nm, M.d_part.as<unsigned long long>(), M.d_tscan.as<unsigned long long>(), c->stream));
        CK(launch_enc_scan(P.nhits, nm, M.d_part.as<unsigned long long>(), M.d_hscan.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(M.ev_c1, c->stream));
        uint64_t *tot = M.h_small.as<uint64_t>();
        CK(cudaMemcpyAsync(tot, M.d_tscan.as<uint64_t>() + nm, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(tot + 1, M.d_hscan.as<uint64_t>() + nm, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(tot + 2, M.d_error.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (uint32_t(tot[2]))
                return fail(c, TRN_ERR_STATE, "a match of the docs pass is not accepted by its query's collect program (internal error)");
        float countMs{0};
        (void)cudaEventElapsedTime(&countMs, M.ev_c0, M.ev_c1);
        const uint64_t nt = tot[0], nh = tot[1];

        // ---- the result's pinned host buffers, sized once
        CK(M.h_term_off.ensure((nm + 1) * 8));
        CK(M.h_terms.ensure(std::max<size_t>(4, nt * 4)));
        CK(M.h_freqs.ensure(std::max<size_t>(4, nt * 4)));
        CK(M.h_hit_off.ensure((nt + 1) * 8));
        CK(M.h_hits.ensure(std::max<size_t>(sizeof(trn_hit), nh * sizeof(trn_hit))));
        CK(cudaMemcpyAsync(M.h_term_off.as<uint64_t>() + nm, M.d_tscan.as<uint64_t>() + nm, 8, cudaMemcpyDeviceToHost, c->stream));
        M.h_hit_off.as<uint64_t>()[nt] = nh;

        // ---- write pass, chunk by chunk of matches: a chunk's terms and hits go through device buffers sized for it
        uint64_t chunk = std::min<uint64_t>(std::max<uint64_t>(1, c->match_chunk), std::max<uint64_t>(1, nm));
        float    writeMs{0};
        uint32_t chunks{0};
        for (uint64_t m0 = 0; m0 < nm;) {
                const uint64_t m1 = std::min(nm, m0 + chunk), n = m1 - m0;
                uint64_t *     sc = tot + 4; // the scans at the chunk's bounds
                CK(cudaMemcpyAsync(sc, M.d_tscan.as<uint64_t>() + m0, 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(sc + 1, M.d_tscan.as<uint64_t>() + m1, 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(sc + 2, M.d_hscan.as<uint64_t>() + m0, 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(sc + 3, M.d_hscan.as<uint64_t>() + m1, 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                const uint64_t t0c = sc[0], ntc = sc[1] - sc[0], h0c = sc[2], nhc = sc[3] - sc[2];
                cudaError_t    e = M.d_term_off.ensure(n * 8);
                for (DevBuf *b : {&M.d_terms, &M.d_freqs})
                        if (e == cudaSuccess)
                                e = b->ensure(std::max<uint64_t>(4, ntc * 4));
                if (e == cudaSuccess)
                        e = M.d_hit_off.ensure(std::max<uint64_t>(8, ntc * 8));
                if (e == cudaSuccess)
                        e = M.d_hits.ensure(std::max<uint64_t>(16, nhc * sizeof(trn_hit)));
                if (e == cudaErrorMemoryAllocation && chunk > 1) { // the chunk's outputs do not fit: halve it
                        (void)cudaGetLastError();
                        chunk = (chunk + 1) / 2;
                        continue;
                }
                CK(e);
                P.m0           = m0;
                P.m1           = m1;
                P.term_base    = t0c;
                P.hit_base     = h0c;
                P.term_offsets = M.d_term_off.as<uint64_t>();
                P.out_terms    = M.d_terms.as<uint32_t>();
                P.out_freqs    = M.d_freqs.as<uint32_t>();
                P.hit_offsets  = M.d_hit_off.as<uint64_t>();
                P.out_hits     = M.d_hits.as<trn_hit>();
                CK(cudaEventRecord(M.ev_w0, c->stream));
                CK(launch_collect_write(P, c->stream));
                CK(cudaEventRecord(M.ev_w1, c->stream));
                CK(cudaMemcpyAsync(M.h_term_off.as<uint64_t>() + m0, P.term_offsets, n * 8, cudaMemcpyDeviceToHost, c->stream));
                if (ntc) {
                        CK(cudaMemcpyAsync(M.h_terms.as<uint32_t>() + t0c, P.out_terms, ntc * 4, cudaMemcpyDeviceToHost, c->stream));
                        CK(cudaMemcpyAsync(M.h_freqs.as<uint32_t>() + t0c, P.out_freqs, ntc * 4, cudaMemcpyDeviceToHost, c->stream));
                        CK(cudaMemcpyAsync(M.h_hit_off.as<uint64_t>() + t0c, P.hit_offsets, ntc * 8, cudaMemcpyDeviceToHost, c->stream));
                }
                if (nhc)
                        CK(cudaMemcpyAsync(M.h_hits.as<trn_hit>() + h0c, P.out_hits, nhc * sizeof(trn_hit), cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream)); // the chunk's device buffers are reused by the next chunk
                float ms{0};
                if (cudaEventElapsedTime(&ms, M.ev_w0, M.ev_w1) == cudaSuccess)
                        writeMs += ms;
                m0 = m1;
                ++chunks;
        }
        CK(cudaEventRecord(M.ev_end, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        c->last_routes     = std::move(routes);
        c->tm.total_ms     = float(now_ms() - t0);
        out->nq            = nq;
        out->total_matches = nm;
        out->total_terms   = nt;
        out->total_hits    = nh;
        out->doc_offsets   = M.h_doc_off.as<uint64_t>();
        out->docids        = M.h_docids.as<uint32_t>();
        out->term_offsets  = M.h_term_off.as<uint64_t>();
        out->terms         = M.h_terms.as<uint32_t>();
        out->freqs         = M.h_freqs.as<uint32_t>();
        out->hit_offsets   = M.h_hit_off.as<uint64_t>();
        out->hits          = M.h_hits.as<trn_hit>();
        out->chunks        = chunks;
        out->count_ms      = countMs;
        out->write_ms      = writeMs;
        float ms{0};
        if (cudaEventElapsedTime(&ms, c->ev0, M.ev_end) == cudaSuccess)
                out->device_ms = ms;
        if (cudaEventElapsedTime(&ms, c->evk0, M.ev_docs) == cudaSuccess)
                out->docs_ms = ms;
        return TRN_OK;
}

static int debug_plan_batch(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                            const trn_query *queries, uint32_t nq, int mode, uint32_t k, BatchPlan &plan, char *err, size_t errcap,
                            GroupStarts *groups = nullptr) {
        auto seterr = [&](const std::string &m, int rc) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return rc;
        };
        if (!index || !terms || !queries || !nq || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || mode < 0 || mode > TRN_MODE_MATCHED_TERMS)
                return seterr("bad arguments", TRN_ERR_ARG);
        BlockDirectory       dir;
        std::vector<DevTerm> ht;
        GroupStarts          gs;
        try {
                build_directory(codec, index, nbytes, terms, nterms, 1, dir);
                ht = dev_terms(dir, terms, nterms);
                if (codec == TRN_CODEC_GOOGLE)
                        gs = group_starts(dir);
        } catch (const std::exception &e) {
                return seterr(e.what(), TRN_ERR_FORMAT);
        }
        PlanConfig pc   = initial_plan_config();
        pc.codec        = codec;
        pc.allow_phrase = codec == TRN_CODEC_GOOGLE;
        docid_span(ht, pc.min_docid, max_docid);
        pc.max_docid            = max_docid;
        const DenseSelection ds = select_dense_terms(pc, ht, nbytes); // what trn_upload_index keeps
        std::string          perr;
        const int            rc = plan_batch(pc, ht, ds.order.empty() ? nullptr : ds.off.data(), queries, nq, mode, k, plan, perr, nullptr,
                                                gs.base.empty() ? nullptr : &gs);
        if (groups)
                *groups = std::move(gs);
        return rc == TRN_OK ? TRN_OK : seterr(perr, rc);
}

extern "C" int trn_debug_plan(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                              const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint8_t *routes, uint32_t *nslots, char *err, size_t errcap) {
        if (!routes || !nslots)
                return TRN_ERR_ARG;
        BatchPlan plan;
        if (const int rc = debug_plan_batch(codec, index, nbytes, terms, nterms, max_docid, queries, nq, mode, k, plan, err, errcap); rc != TRN_OK)
                return rc;
        for (uint32_t q = 0; q < nq; ++q)
                routes[q] = uint8_t(plan.queries[q].route);
        nslots[0] = plan.nslots;
        nslots[1] = plan.tree_slots;
        return TRN_OK;
}

// trn_debug_dense_runs / trn_debug_mixed_runs / trn_debug_cand_runs: the run tickets of BatchPlan::dense_runs, mixed_runs or cand_runs
enum class RunTickets { dense, mixed, cand };
static int debug_run_tickets(RunTickets which, int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                             const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n,
                             char *err, size_t errcap) {
        if (!qtiles || !n)
                return TRN_ERR_ARG;
        BatchPlan   plan;
        GroupStarts gs; // the first docID of every lead group (the third word of a candidate ticket)
        if (const int rc = debug_plan_batch(codec, index, nbytes, terms, nterms, max_docid, queries, nq, mode, k, plan, err, errcap, &gs); rc != TRN_OK)
                return rc;
        for (uint32_t q = 0; q < nq; ++q) {
                qtiles[2 * q]     = plan.queries[q].tile_lo;
                qtiles[2 * q + 1] = plan.queries[q].ntiles;
        }
        const std::vector<uint2> &runs = which == RunTickets::mixed ? plan.mixed_runs : which == RunTickets::cand ? plan.cand_runs : plan.dense_runs;
        *n                             = runs.size();
        if (cap < *n)
                return TRN_ERR_CAPACITY;
        for (uint64_t t = 0; t < *n; ++t) {
                const uint2     e  = runs[t];
                const DevQuery &dq = plan.queries[e.x];
                tickets[3 * t]     = e.x;
                tickets[3 * t + 1] = e.y;
                tickets[3 * t + 2] = which == RunTickets::cand ? gs.first[gs.base[plan.steps[dq.step_begin].term] + e.y]
                                                               : dense_run_end(e.y, dq.tile_lo, dq.ntiles, plan.exec_shift);
        }
        return TRN_OK;
}

extern "C" int trn_debug_dense_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                                    const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n,
                                    char *err, size_t errcap) {
        return debug_run_tickets(RunTickets::dense, codec, index, nbytes, terms, nterms, max_docid, queries, nq, mode, k, qtiles, tickets, cap, n, err, errcap);
}

extern "C" int trn_debug_mixed_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                                    const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n,
                                    char *err, size_t errcap) {
        return debug_run_tickets(RunTickets::mixed, codec, index, nbytes, terms, nterms, max_docid, queries, nq, mode, k, qtiles, tickets, cap, n, err, errcap);
}

extern "C" int trn_debug_cand_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                                   const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n,
                                   char *err, size_t errcap) {
        return debug_run_tickets(RunTickets::cand, codec, index, nbytes, terms, nterms, max_docid, queries, nq, mode, k, qtiles, tickets, cap, n, err, errcap);
}

// trn_debug_dense_terms / trn_debug_probe_terms: the selection of one tier of resident bitmaps
static int debug_bitmap_terms(bool probe, int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t *offsets,
                              uint32_t *nselected, uint64_t *bitmap_bytes, char *err, size_t errcap) {
        auto seterr = [&](const std::string &m, int rc) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return rc;
        };
        if (!index || !terms || (nterms && !offsets) || !nselected || !bitmap_bytes || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return seterr("bad arguments", TRN_ERR_ARG);
        DenseSelection s;
        try {
                BlockDirectory dir;
                build_directory(codec, index, nbytes, terms, nterms, 1, dir);
                PlanConfig pc = initial_plan_config();
                pc.codec      = codec;
                const std::vector<DevTerm> ht = dev_terms(dir, terms, nterms);
                s                             = select_dense_terms(pc, ht, nbytes);
                if (probe)
                        s = select_probe_terms(pc, ht, nbytes, s);
        } catch (const std::exception &e) {
                return seterr(e.what(), TRN_ERR_FORMAT);
        }
        if (nterms)
                std::memcpy(offsets, s.off.data(), nterms * 4);
        *nselected    = uint32_t(s.order.size());
        *bitmap_bytes = s.words * 4;
        return TRN_OK;
}

extern "C" int trn_debug_dense_terms(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t *offsets,
                                     uint32_t *nselected, uint64_t *bitmap_bytes, char *err, size_t errcap) {
        return debug_bitmap_terms(false, codec, index, nbytes, terms, nterms, offsets, nselected, bitmap_bytes, err, errcap);
}

extern "C" int trn_debug_probe_terms(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t *offsets,
                                     uint32_t *nselected, uint64_t *bitmap_bytes, char *err, size_t errcap) {
        return debug_bitmap_terms(true, codec, index, nbytes, terms, nterms, offsets, nselected, bitmap_bytes, err, errcap);
}

extern "C" int trn_debug_dense_bitmap(trn_ctx *c, uint32_t term, uint32_t *out, uint64_t cap, uint64_t *base, uint64_t *nwords) {
        if (!c || !base || !nwords)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (term >= c->nterms)
                return fail(c, TRN_ERR_ARG, "trn_debug_dense_bitmap: no such term");
        *base   = 0;
        *nwords = 0;
        if (!c->dense_terms || c->h_dense_off[term] == kDenseNone)
                return TRN_OK;
        dense_span(c->h_terms[term], *base, *nwords);
        if (cap < *nwords || !out)
                return fail(c, TRN_ERR_CAPACITY, "trn_debug_dense_bitmap: buffer too small");
        CK(cudaSetDevice(c->device));
        CK(cudaMemcpy(out, c->d_dense.as<uint32_t>() + c->h_dense_off[term], *nwords * 4, cudaMemcpyDeviceToHost));
        return TRN_OK;
}

extern "C" int trn_last_timings(trn_ctx *c, trn_timings *out) {
        if (!c || !out)
                return TRN_ERR_ARG;
        *out = c->tm;
        return TRN_OK;
}

extern "C" int trn_last_topk_device(trn_ctx *c, void **docids, void **scores, void **counts) {
        if (!c)
                return TRN_ERR_ARG;
        if (c->last_mode != TRN_MODE_SCORED_TOPK)
                return fail(c, TRN_ERR_STATE, "last batch was not SCORED_TOPK");
        if (docids)
                *docids = c->d_topk_docids.p;
        if (scores)
                *scores = c->d_topk_scores.p;
        if (counts)
                *counts = c->d_topk_counts.p;
        return TRN_OK;
}

extern "C" int trn_merge_topk(trn_ctx *c, const void *docids, const void *scores, uint32_t nshards, uint32_t nq, uint32_t k, void *out_docids, void *out_scores) {
        if (!c || !docids || !scores || !out_docids || !out_scores || !nshards || !nq || !k || k > kernel_max_k())
                return c ? fail(c, TRN_ERR_ARG, "trn_merge_topk: bad arguments") : TRN_ERR_ARG;
        CK(cudaSetDevice(c->device));
        CK(launch_topk_merge(static_cast<const uint32_t *>(docids), static_cast<const float *>(scores), nshards, nq, k, static_cast<uint32_t *>(out_docids),
                             static_cast<float *>(out_scores), c->stream));
        return TRN_OK;
}

// =================================================================================================== device-side encoder (GOOGLE)
// Term-major postings resident in HBM, in the layout the encode kernels read: trn_encode_google / trn_encode_lucene upload the caller's,
// trn_index_documents builds them on the device.  h_term_begin = the host's copy of term_begin (block and unit numbering is host work).
struct DevPostings {
        const uint64_t *          h_term_begin;
        uint32_t                  nterms;
        const unsigned long long *term_begin;
        const uint32_t *          docids, *freqs, *positions; // positions null: 1..freq
        const uint8_t *           plens = nullptr;            // per hit: payload bytes (null: no payloads; needs positions)
        const unsigned long long *payloads = nullptr;         // per hit: the payload in its low plens[] bytes
};

// The encode itself: sizes, scans and the write over device-resident postings; the chunks stay in d_out.  chunk[t] / toff[t] = bytes and
// offset of term t's chunk, *out_bytes their total (set before the capacity refusals, as trn_encode_google documents), *nblocks the blocks
// committed (the countdown's advance).  cap = the caller's buffer (have_out false: none).
static int encode_google_device(trn_ctx *c, const DevPostings &P, uint32_t block_docs, uint32_t skiplist_step, uint32_t phase0, bool have_out, uint64_t cap,
                                uint64_t *out_bytes, DevBuf &d_out, std::vector<uint64_t> &chunk, std::vector<uint64_t> &toff, uint64_t *nblocks_out,
                                float *device_ms) {
        const uint64_t *const term_begin = P.h_term_begin;
        const uint32_t        nterms     = P.nterms;
        const uint64_t        nposts     = term_begin[nterms];
        const bool            positions  = P.positions != nullptr;
        std::vector<uint64_t> blk_begin(nterms + 1);
        uint64_t              nblocks{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                blk_begin[t] = nblocks;
                nblocks += (term_begin[t + 1] - term_begin[t] + block_docs - 1) / block_docs;
        }
        blk_begin[nterms] = nblocks;
        DevBuf   d_bb, d_hb, d_bsz, d_bterm, d_boff, d_part, d_toff, d_cb, d_err;
        const size_t parts = size_t(std::max(nposts, nblocks) / 4096 + 4);
        CK(d_bb.ensure((size_t(nterms) + 1) * 8));
        CK(d_bsz.ensure(std::max<size_t>(4, nblocks * 4)));
        CK(d_bterm.ensure(std::max<size_t>(4, nblocks * 4)));
        CK(d_boff.ensure((nblocks + 1) * 8));
        CK(d_part.ensure(parts * 8));
        CK(d_toff.ensure((size_t(nterms) + 1) * 8));
        CK(d_cb.ensure(size_t(nterms) * 8));
        CK(d_err.ensure(4));
        CK(cudaMemcpyAsync(d_bb.p, blk_begin.data(), (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        if (positions)
                CK(d_hb.ensure((nposts + 1) * 8));
        CK(cudaMemsetAsync(d_err.p, 0, 4, c->stream));
        EncParams E{};
        E.term_begin    = P.term_begin;
        E.blk_begin     = d_bb.as<unsigned long long>();
        E.nterms        = nterms;
        E.nblocks       = nblocks;
        E.docids        = P.docids;
        E.freqs         = P.freqs;
        E.positions     = P.positions;
        E.hit_begin     = positions ? d_hb.as<unsigned long long>() : nullptr;
        E.block_docs    = block_docs;
        E.skiplist_step = skiplist_step;
        E.phase0        = phase0;
        E.bsz           = d_bsz.as<uint32_t>();
        E.bterm         = d_bterm.as<uint32_t>();
        E.boff          = d_boff.as<unsigned long long>();
        E.term_off      = d_toff.as<unsigned long long>();
        E.error         = d_err.as<uint32_t>();
        cudaEvent_t e0 = c->ev0, e1 = c->ev1, e2 = c->evk0, e3 = c->evk1;
        CK(cudaEventRecord(e0, c->stream));
        if (positions)
                CK(launch_enc_scan(P.freqs, nposts, d_part.as<unsigned long long>(), d_hb.as<unsigned long long>(), c->stream));
        CK(launch_enc_google_sizes(E, EncPayloads{P.plens, P.payloads}, c->stream));
        CK(launch_enc_scan(d_bsz.as<uint32_t>(), nblocks, d_part.as<unsigned long long>(), d_boff.as<unsigned long long>(), c->stream));
        CK(launch_enc_term_sizes(E, d_cb.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(e1, c->stream));
        // chunk offsets: a prefix sum over the terms on the host (the output size must be known here anyway)
        chunk.assign(nterms, 0);
        toff.assign(size_t(nterms) + 1, 0);
        uint32_t herr{0};
        CK(cudaMemcpyAsync(chunk.data(), d_cb.p, size_t(nterms) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&herr, d_err.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (herr)
                return fail(c, TRN_ERR_ARG, P.plens ? "google encoder: document IDs must be > 0 and strictly ascending, positions in 1..16383 (0 only with a payload) "
                                                      "and non-decreasing, payloads of at most 8 bytes"
                                                    : "google encoder: document IDs must be > 0 and strictly ascending, positions in 1..16383 and non-decreasing");
        uint64_t total{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                toff[t] = total;
                total += chunk[t];
        }
        toff[nterms] = total;
        *out_bytes   = total;
        if (total >= (1ull << 32))
                return fail(c, TRN_ERR_CAPACITY, "google encoder: the index of one source is limited to 4 GiB (range32_t, codecs.h:17-55)");
        if (total > cap || !have_out)
                return fail(c, TRN_ERR_CAPACITY, "trn_encode_google: output buffer too small");
        CK(d_out.ensure(std::max<size_t>(4, total)));
        E.out = d_out.as<uint8_t>();
        CK(cudaMemcpyAsync(d_toff.p, toff.data(), (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaEventRecord(e2, c->stream));
        CK(cudaMemsetAsync(d_out.p, 0, std::max<size_t>(4, total), c->stream)); // a term without documents is its zero u16
        CK(launch_enc_google_write(E, EncPayloads{P.plens, P.payloads}, c->stream));
        CK(cudaEventRecord(e3, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        *nblocks_out = nblocks;
        if (device_ms) {
                float a{0}, b{0};
                CK(cudaEventElapsedTime(&a, e0, e1));
                CK(cudaEventElapsedTime(&b, e2, e3));
                *device_ms = a + b;
        }
        c->have_kernel_events = false;
        return TRN_OK;
}

extern "C" int trn_encode_google_payloads(trn_ctx *c, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs,
                                          const uint32_t *positions, const uint8_t *payload_lens, const uint64_t *payloads, uint32_t block_docs,
                                          uint32_t skiplist_step, uint32_t *countdown, uint8_t *out, uint64_t cap, uint64_t *out_bytes, trn_term *terms,
                                          float *device_ms) {
        if (!c)
                return TRN_ERR_ARG;
        if (!term_begin || !nterms || !out_bytes || !terms || block_docs == 0 || block_docs > 128 || skiplist_step == 0 ||
            (countdown && (*countdown == 0 || *countdown > skiplist_step)))
                return fail(c, TRN_ERR_ARG, "trn_encode_google: bad arguments");
        if (!payload_lens != !payloads || (payload_lens && !positions))
                return fail(c, TRN_ERR_ARG, "trn_encode_google_payloads: payload_lens and payloads are given together, and with positions");
        const uint64_t nposts = term_begin[nterms];
        if (term_begin[0] != 0 || (nposts && (!docids || !freqs)))
                return fail(c, TRN_ERR_ARG, "trn_encode_google: bad arguments");
        CK(cudaSetDevice(c->device));
        for (uint32_t t = 0; t < nterms; ++t)
                if (term_begin[t + 1] < term_begin[t] || term_begin[t + 1] - term_begin[t] > 0xffffffffull)
                        return fail(c, TRN_ERR_ARG, "trn_encode_google: term_begin must ascend (at most 2^32 - 1 documents per term)");
        uint64_t nhits{0};
        if (positions)
                for (uint64_t i = 0; i < nposts; ++i)
                        nhits += freqs[i];
        const uint32_t phase0 = countdown ? (skiplist_step - *countdown) % skiplist_step : 0u;
        DevBuf         d_tb, d_doc, d_fr, d_pos, d_out;
        CK(d_tb.ensure((size_t(nterms) + 1) * 8));
        CK(d_doc.ensure(std::max<size_t>(4, nposts * 4)));
        CK(d_fr.ensure(std::max<size_t>(4, nposts * 4)));
        CK(cudaMemcpyAsync(d_tb.p, term_begin, (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        if (nposts) {
                CK(cudaMemcpyAsync(d_doc.p, docids, nposts * 4, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_fr.p, freqs, nposts * 4, cudaMemcpyHostToDevice, c->stream));
        }
        if (positions) {
                CK(d_pos.ensure(std::max<size_t>(4, nhits * 4)));
                if (nhits)
                        CK(cudaMemcpyAsync(d_pos.p, positions, nhits * 4, cudaMemcpyHostToDevice, c->stream));
        }
        DevBuf   d_pl, d_pv;
        if (payload_lens) {
                CK(d_pl.ensure(std::max<size_t>(4, nhits)));
                CK(d_pv.ensure(std::max<size_t>(8, nhits * 8)));
                if (nhits) {
                        CK(cudaMemcpyAsync(d_pl.p, payload_lens, nhits, cudaMemcpyHostToDevice, c->stream));
                        CK(cudaMemcpyAsync(d_pv.p, payloads, nhits * 8, cudaMemcpyHostToDevice, c->stream));
                }
        }
        DevPostings P{term_begin, nterms, d_tb.as<unsigned long long>(), d_doc.as<uint32_t>(), d_fr.as<uint32_t>(), positions ? d_pos.as<uint32_t>() : nullptr};
        if (payload_lens) {
                P.plens    = d_pl.as<uint8_t>();
                P.payloads = d_pv.as<unsigned long long>();
        }
        std::vector<uint64_t> chunk, toff;
        uint64_t              nblocks{0};
        if (const int r = encode_google_device(c, P, block_docs, skiplist_step, phase0, out != nullptr, cap, out_bytes, d_out, chunk, toff, &nblocks, device_ms))
                return r;
        CK(cudaMemcpyAsync(out, d_out.p, *out_bytes, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        for (uint32_t t = 0; t < nterms; ++t) {
                terms[t].documents = uint32_t(term_begin[t + 1] - term_begin[t]);
                terms[t].chunk_off = uint32_t(toff[t]);
                terms[t].chunk_len = uint32_t(chunk[t]);
        }
        if (countdown)
                *countdown = skiplist_step - uint32_t((uint64_t(phase0) + nblocks) % skiplist_step);
        return TRN_OK;
}

extern "C" int trn_encode_google(trn_ctx *c, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                                 uint32_t block_docs, uint32_t skiplist_step, uint32_t *countdown, uint8_t *out, uint64_t cap, uint64_t *out_bytes, trn_term *terms,
                                 float *device_ms) {
        return trn_encode_google_payloads(c, term_begin, nterms, docids, freqs, positions, nullptr, nullptr, block_docs, skiplist_step, countdown, out, cap, out_bytes,
                                          terms, device_ms);
}

// =================================================================================================== device-side encoder (LUCENE)
// The encode itself over device-resident postings; index and hits.data stay in d_iout / d_hout.  toff[t] = offset of term t's chunk
// (nterms + 1), *index_bytes / *hits_bytes the totals (set before the capacity refusals).  have_index / have_hits: the caller has buffers.
static int encode_lucene_device(trn_ctx *c, const DevPostings &P, bool have_index, uint64_t index_cap, uint64_t *index_bytes, bool have_hits, uint64_t hits_cap,
                                uint64_t *hits_bytes, DevBuf &d_iout, DevBuf &d_hout, std::vector<uint64_t> &toff, float *device_ms,
                                std::vector<uint64_t> *hits_toff = nullptr) {
        const uint64_t *const term_begin = P.h_term_begin;
        const uint32_t        nterms     = P.nterms;
        const uint64_t        nposts     = term_begin[nterms];
        constexpr uint32_t N = Codecs::Lucene::BLOCK_SIZE;
        // doc units: every term's full blocks, then its tail; the chunk headers and skiplists around them are fixed by the block counts
        std::vector<uint64_t> dunit(nterms + 1), fixed(nterms + 1), hunit(nterms + 1), th(nterms + 1);
        uint64_t              ndunits{0}, fx{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                const uint64_t nfull = (term_begin[t + 1] - term_begin[t]) / N;
                dunit[t]             = ndunits;
                fixed[t]             = fx;
                ndunits += nfull + 1u;
                fx += 14u + 22u * std::min<uint64_t>(nfull, 65535u);
        }
        dunit[nterms] = ndunits;
        fixed[nterms] = fx;
        DevBuf   d_du, d_hu, d_fx, d_hb, d_th, d_dsz, d_hsz, d_dterm, d_hterm, d_doff, d_hoff, d_part, d_toff, d_hto, d_err;
        const size_t tw = (size_t(nterms) + 1) * 8;
        CK(d_du.ensure(tw));
        CK(d_hu.ensure(tw));
        CK(d_fx.ensure(tw));
        CK(d_th.ensure(tw));
        CK(d_toff.ensure(tw));
        CK(d_hto.ensure(tw));
        CK(d_hb.ensure((nposts + 1) * 8));
        CK(d_dsz.ensure(ndunits * 4));
        CK(d_dterm.ensure(ndunits * 4));
        CK(d_doff.ensure((ndunits + 1) * 8));
        CK(d_err.ensure(4));
        CK(cudaMemcpyAsync(d_du.p, dunit.data(), tw, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_fx.p, fixed.data(), tw, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemsetAsync(d_err.p, 0, 4, c->stream));
        // (1) hits of every posting (scan of the freqs) and of every term; the host needs the per-term totals to number the hit units
        CK(d_part.ensure(size_t(std::max(nposts, ndunits) / 4096 + 4) * 8));
        float          ms{0}, a{0};
        cudaEvent_t    e0 = c->ev0, e1 = c->ev1;
        CK(cudaEventRecord(e0, c->stream));
        CK(launch_enc_scan(P.freqs, nposts, d_part.as<unsigned long long>(), d_hb.as<unsigned long long>(), c->stream));
        CK(launch_enc_lucene_term_hits(P.term_begin, d_hb.as<unsigned long long>(), nterms, d_th.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(e1, c->stream));
        CK(cudaMemcpyAsync(th.data(), d_th.p, tw, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&a, e0, e1));
        ms += a;
        uint64_t nhunits{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                hunit[t] = nhunits;
                nhunits += (th[t + 1] - th[t]) / N + 1u;
        }
        hunit[nterms]       = nhunits;
        const uint64_t nhits = th[nterms];
        CK(d_hsz.ensure(nhunits * 4));
        CK(d_hterm.ensure(nhunits * 4));
        CK(d_hoff.ensure((nhunits + 1) * 8));
        CK(d_part.ensure(size_t(nhunits / 4096 + 4) * 8));
        CK(cudaMemcpyAsync(d_hu.p, hunit.data(), tw, cudaMemcpyHostToDevice, c->stream));
        EncLuceneParams E{};
        E.term_begin  = P.term_begin;
        E.dunit_begin = d_du.as<unsigned long long>();
        E.hunit_begin = d_hu.as<unsigned long long>();
        E.nterms      = nterms;
        E.ndunits     = ndunits;
        E.nhunits     = nhunits;
        E.docids      = P.docids;
        E.freqs       = P.freqs;
        E.positions   = nhits ? P.positions : nullptr;
        E.hit_begin   = d_hb.as<unsigned long long>();
        E.dsz         = d_dsz.as<uint32_t>();
        E.hsz         = d_hsz.as<uint32_t>();
        E.dterm       = d_dterm.as<uint32_t>();
        E.hterm       = d_hterm.as<uint32_t>();
        E.doff        = d_doff.as<unsigned long long>();
        E.hoff        = d_hoff.as<unsigned long long>();
        E.term_off    = d_toff.as<unsigned long long>();
        E.error       = d_err.as<uint32_t>();
        const EncPayloads pay{nhits ? P.plens : nullptr, nhits ? P.payloads : nullptr};
        // (2) sizes of every unit, their scans, the chunk and hits.data offsets of every term
        CK(cudaEventRecord(e0, c->stream));
        CK(launch_enc_lucene_sizes(E, pay, c->stream));
        CK(launch_enc_scan(d_dsz.as<uint32_t>(), ndunits, d_part.as<unsigned long long>(), d_doff.as<unsigned long long>(), c->stream));
        CK(launch_enc_scan(d_hsz.as<uint32_t>(), nhunits, d_part.as<unsigned long long>(), d_hoff.as<unsigned long long>(), c->stream));
        CK(launch_enc_lucene_terms(E, d_fx.as<unsigned long long>(), d_toff.as<unsigned long long>(), d_hto.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(e1, c->stream));
        std::vector<uint64_t> hto(nterms + 1);
        uint32_t              herr{0};
        toff.assign(size_t(nterms) + 1, 0);
        CK(cudaMemcpyAsync(toff.data(), d_toff.p, tw, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(hto.data(), d_hto.p, tw, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&herr, d_err.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&a, e0, e1));
        ms += a;
        if (herr)
                return fail(c, TRN_ERR_ARG, pay.plens ? "lucene encoder: document IDs must be > 0 and strictly ascending, positions in 1..16383 (0 only with a payload) "
                                                      "and non-decreasing, payloads of at most 8 bytes"
                                                    : "lucene encoder: document IDs must be > 0 and strictly ascending, positions in 1..16383 and non-decreasing");
        const uint64_t total = toff[nterms], htotal = hto[nterms];
        *index_bytes         = total;
        *hits_bytes          = htotal;
        if (total >= (1ull << 32) || htotal >= (1ull << 32))
                return fail(c, TRN_ERR_CAPACITY, "lucene encoder: the index and hits.data of one source are limited to 4 GiB (u32 chunk and hits offsets)");
        if (total > index_cap || htotal > hits_cap || !have_index || (htotal && !have_hits))
                return fail(c, TRN_ERR_CAPACITY, "trn_encode_lucene: output buffer too small");
        CK(d_iout.ensure(std::max<size_t>(4, total)));
        CK(d_hout.ensure(std::max<size_t>(4, htotal)));
        E.index_out = d_iout.as<uint8_t>();
        E.hits_out  = d_hout.as<uint8_t>();
        // (3) the bytes: every byte of both outputs is written by exactly one unit's warp
        CK(cudaEventRecord(e0, c->stream));
        CK(launch_enc_lucene_write(E, pay, c->stream));
        CK(cudaEventRecord(e1, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&a, e0, e1));
        ms += a;
        if (device_ms)
                *device_ms = ms;
        if (hits_toff)
                hits_toff->swap(hto);
        c->have_kernel_events = false;
        return TRN_OK;
}

extern "C" int trn_encode_lucene_payloads(trn_ctx *c, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs,
                                          const uint32_t *positions, const uint8_t *payload_lens, const uint64_t *payloads, uint8_t *index_out, uint64_t index_cap,
                                          uint64_t *index_bytes, uint8_t *hits_out, uint64_t hits_cap, uint64_t *hits_bytes, trn_term *terms, float *device_ms) {
        if (!c)
                return TRN_ERR_ARG;
        if (!term_begin || !nterms || !index_bytes || !hits_bytes || !terms)
                return fail(c, TRN_ERR_ARG, "trn_encode_lucene: bad arguments");
        if (!payload_lens != !payloads || (payload_lens && !positions))
                return fail(c, TRN_ERR_ARG, "trn_encode_lucene_payloads: payload_lens and payloads are given together, and with positions");
        const uint64_t nposts = term_begin[nterms];
        if (term_begin[0] != 0 || (nposts && (!docids || !freqs)))
                return fail(c, TRN_ERR_ARG, "trn_encode_lucene: bad arguments");
        for (uint32_t t = 0; t < nterms; ++t)
                if (term_begin[t + 1] < term_begin[t] || term_begin[t + 1] - term_begin[t] > 0xffffffffull)
                        return fail(c, TRN_ERR_ARG, "trn_encode_lucene: term_begin must ascend (at most 2^32 - 1 documents per term)");
        uint64_t nhits{0};
        if (positions)
                for (uint64_t i = 0; i < nposts; ++i)
                        nhits += freqs[i];
        CK(cudaSetDevice(c->device));
        DevBuf   d_tb, d_doc, d_fr, d_pos, d_iout, d_hout;
        const size_t tw = (size_t(nterms) + 1) * 8;
        CK(d_tb.ensure(tw));
        CK(d_doc.ensure(std::max<size_t>(4, nposts * 4)));
        CK(d_fr.ensure(std::max<size_t>(4, nposts * 4)));
        CK(cudaMemcpyAsync(d_tb.p, term_begin, tw, cudaMemcpyHostToDevice, c->stream));
        if (nposts) {
                CK(cudaMemcpyAsync(d_doc.p, docids, nposts * 4, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_fr.p, freqs, nposts * 4, cudaMemcpyHostToDevice, c->stream));
        }
        if (nhits) {
                CK(d_pos.ensure(nhits * 4));
                CK(cudaMemcpyAsync(d_pos.p, positions, nhits * 4, cudaMemcpyHostToDevice, c->stream));
        }
        DevBuf   d_pl, d_pv;
        DevPostings P{term_begin, nterms, d_tb.as<unsigned long long>(), d_doc.as<uint32_t>(), d_fr.as<uint32_t>(), nhits ? d_pos.as<uint32_t>() : nullptr};
        if (payload_lens && nhits) {
                CK(d_pl.ensure(nhits));
                CK(d_pv.ensure(nhits * 8));
                CK(cudaMemcpyAsync(d_pl.p, payload_lens, nhits, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_pv.p, payloads, nhits * 8, cudaMemcpyHostToDevice, c->stream));
                P.plens    = d_pl.as<uint8_t>();
                P.payloads = d_pv.as<unsigned long long>();
        }
        std::vector<uint64_t> toff;
        if (const int r = encode_lucene_device(c, P, index_out != nullptr, index_cap, index_bytes, hits_out != nullptr, hits_cap, hits_bytes, d_iout, d_hout, toff, device_ms))
                return r;
        CK(cudaMemcpyAsync(index_out, d_iout.p, *index_bytes, cudaMemcpyDeviceToHost, c->stream));
        if (*hits_bytes)
                CK(cudaMemcpyAsync(hits_out, d_hout.p, *hits_bytes, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        for (uint32_t t = 0; t < nterms; ++t) {
                terms[t].documents = uint32_t(term_begin[t + 1] - term_begin[t]);
                terms[t].chunk_off = uint32_t(toff[t]);
                terms[t].chunk_len = uint32_t(toff[t + 1] - toff[t]);
        }
        return TRN_OK;
}

extern "C" int trn_encode_lucene(trn_ctx *c, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                                 uint8_t *index_out, uint64_t index_cap, uint64_t *index_bytes, uint8_t *hits_out, uint64_t hits_cap, uint64_t *hits_bytes,
                                 trn_term *terms, float *device_ms) {
        return trn_encode_lucene_payloads(c, term_begin, nterms, docids, freqs, positions, nullptr, nullptr, index_out, index_cap, index_bytes, hits_out, hits_cap,
                                          hits_bytes, terms, device_ms);
}

// =================================================================================================== indexer
// == SegmentIndexSession begin / insert / commit for one batch of documents (indexer.cpp:14-153, 311-564): the doc-major -> term-major
// inversion is a keys-only radix sort on the device (index_docs.cuh), its output feeds the device encoders without a host round trip.
namespace {
struct IndexPass {
        uint32_t shift, bits;
};
// the passes of the LSD sort over the key bits that can be non-zero (`active`): groups of up to 8 bits starting at an active bit and ending
// at one; a digit that is constant over all keys is never sorted by
std::vector<IndexPass> plan_radix_passes(uint64_t active) {
        std::vector<IndexPass> v;
        for (uint32_t b = 0; b < 64;) {
                if (!((active >> b) & 1u)) {
                        ++b;
                        continue;
                }
                uint32_t bits = std::min(8u, 64u - b);
                while (bits > 1 && !((active >> (b + bits - 1)) & 1u))
                        --bits;
                v.push_back({b, bits});
                b += bits;
        }
        return v;
}
uint64_t low_bits_for(uint64_t maxv) { // mask of the bits the values 0 .. maxv use
        uint32_t b = 0;
        while (b < 64 && (maxv >> b))
                ++b;
        return b == 64 ? ~0ull : (1ull << b) - 1;
}
} // namespace

// working memory of the indexer: an allocation failure is a refusal (split the batch), not a CUDA error
#define CKM(call)                                                                                                                                              \
        do {                                                                                                                                                   \
                cudaError_t e__ = (call);                                                                                                                      \
                if (e__ == cudaErrorMemoryAllocation) {                                                                                                        \
                        cudaGetLastError();                                                                                                                    \
                        return fail(c, TRN_ERR_CAPACITY, "trn_index_documents: working memory cannot be allocated on the device; split the batch");           \
                }                                                                                                                                              \
                if (e__ != cudaSuccess) {                                                                                                                      \
                        c->err = std::string(#call) + ": " + cudaGetErrorString(e__);                                                                          \
                        return TRN_ERR_CUDA;                                                                                                                   \
                }                                                                                                                                              \
        } while (0)

// sorts n keys by the planned passes; the result is in *sorted (a or b).  va / vb (may be null): a u32 per key that moves with it, the
// result in *vsorted.  No host synchronisation.
static int index_radix_sort(trn_ctx *c, DevBuf &a, DevBuf &b, uint64_t n, const std::vector<IndexPass> &passes, DevBuf &counts, DevBuf &part, DevBuf &offs,
                            unsigned long long **sorted, DevBuf *va = nullptr, DevBuf *vb = nullptr, uint32_t **vsorted = nullptr) {
        const uint64_t ntiles = (n + 4095) / 4096;
        uint32_t       maxbits{1};
        for (const auto &p : passes)
                maxbits = std::max(maxbits, p.bits);
        const uint64_t ncounts = (uint64_t(1) << maxbits) * ntiles;
        CKM(counts.ensure(ncounts * 4));
        CKM(offs.ensure((ncounts + 1) * 8));
        CKM(part.ensure((ncounts / 4096 + 4) * 8));
        unsigned long long *in = a.as<unsigned long long>(), *out = b.as<unsigned long long>();
        uint32_t *          vin = va ? va->as<uint32_t>() : nullptr, *vout = va ? vb->as<uint32_t>() : nullptr;
        for (const auto &p : passes) {
                CK(launch_radix_pass(in, out, n, p.shift, p.bits, counts.as<uint32_t>(), part.as<unsigned long long>(), offs.as<unsigned long long>(), c->stream, vin,
                                     vout));
                std::swap(in, out);
                std::swap(vin, vout);
        }
        *sorted = in;
        if (vsorted)
                *vsorted = vin;
        return TRN_OK;
}

extern "C" int trn_index_documents_payloads(trn_ctx *c, int codec, const uint32_t *docids, const uint64_t *doc_offsets, const uint32_t *tokens,
                                            const uint32_t *positions, const uint8_t *payload_lens, const uint64_t *payloads, uint32_t ndocs, uint32_t nterms,
                                            trn_indexed *out) {
        if (!c)
                return TRN_ERR_ARG;
        const double t_begin = now_ms();
        if (!docids || !doc_offsets || !out || !ndocs || !nterms || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || doc_offsets[0] != 0)
                return fail(c, TRN_ERR_ARG, "trn_index_documents: bad arguments");
        if (!payload_lens != !payloads)
                return fail(c, TRN_ERR_ARG, "trn_index_documents_payloads: payload_lens and payloads are given together");
        if (nterms > kIndexMaxTerms)
                return fail(c, TRN_ERR_ARG, "trn_index_documents: " + std::to_string(nterms) + " terms: at most 2^24 per call");
        if (ndocs > kIndexMaxDocs)
                return fail(c, TRN_ERR_ARG, "trn_index_documents: " + std::to_string(ndocs) + " documents: at most 2^26 per call");
        uint64_t maxlen{0};
        uint32_t docs_cnt{0}, max_docid{0};
        for (uint32_t d = 0; d < ndocs; ++d) {
                if (doc_offsets[d + 1] < doc_offsets[d])
                        return fail(c, TRN_ERR_ARG, "trn_index_documents: document " + std::to_string(d) + ": doc_offsets must ascend");
                const uint64_t len = doc_offsets[d + 1] - doc_offsets[d];
                if (!positions && len > 16383u)
                        return fail(c, TRN_ERR_ARG, "trn_index_documents: document " + std::to_string(d) + " (docID " + std::to_string(docids[d]) + "): " +
                                                        std::to_string(len) + " tokens: positions must be below 16384 (Limits::MaxPosition)");
                maxlen = std::max(maxlen, len);
                docs_cnt += len != 0;
                max_docid = std::max(max_docid, docids[d]);
        }
        const uint64_t ntok = doc_offsets[ndocs];
        if (ntok && !tokens)
                return fail(c, TRN_ERR_ARG, "trn_index_documents: bad arguments");
        const bool with_payloads = payload_lens && ntok;
        if (with_payloads && ntok > 0xffffffffull) // the ordinal the sort moves beside every key is a u32
                return fail(c, TRN_ERR_CAPACITY, "trn_index_documents_payloads: " + std::to_string(ntok) + " tokens: at most 2^32 - 1 per call with payloads; split the batch");
        CK(cudaSetDevice(c->device));
        auto &X = c->ix;
        for (auto &e : X.ev)
                if (!e)
                        CK(cudaEventCreate(&e.h));
        const auto doc_of_token = [&](uint64_t i) { return uint32_t(std::upper_bound(doc_offsets, doc_offsets + ndocs + 1, i) - doc_offsets) - 1u; };
        const auto who          = [&](uint32_t d) { return "trn_index_documents: document " + std::to_string(d) + " (docID " + std::to_string(docids[d]) + "): "; };

        DevBuf   d_docids, d_doff, d_tok, d_pos, d_ka, d_kb, d_rank, d_docid_of, d_err, d_counts, d_part, d_offs, d_pflag, d_tflag, d_pscan, d_tscan, d_pbegin, d_tb, d_order,
            d_odoc, d_ofreq, d_opos, d_docterms, d_out, d_hout, d_pl, d_pv, d_va, d_vb, d_opl, d_opv;
        uint64_t herr[IDX_ERR_KINDS];
        // ---- documents: ranks in docID order, docID 0 and duplicates
        CKM(d_docids.ensure(size_t(ndocs) * 4));
        CKM(d_doff.ensure((size_t(ndocs) + 1) * 8));
        CKM(d_ka.ensure(std::max<uint64_t>(ndocs, ntok) * 8));
        CKM(d_kb.ensure(std::max<uint64_t>(ndocs, ntok) * 8));
        CKM(d_rank.ensure(size_t(ndocs) * 4));
        CKM(d_docid_of.ensure(size_t(ndocs) * 4));
        CKM(d_err.ensure(sizeof herr));
        CKM(d_tok.ensure(std::max<uint64_t>(1, ntok) * 4));
        if (positions)
                CKM(d_pos.ensure(std::max<uint64_t>(1, ntok) * 4));
        if (with_payloads) {
                CKM(d_pl.ensure(ntok));
                CKM(d_pv.ensure(ntok * 8));
                CKM(d_va.ensure(ntok * 4));
                CKM(d_vb.ensure(ntok * 4));
                CK(cudaMemcpyAsync(d_pl.p, payload_lens, ntok, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_pv.p, payloads, ntok * 8, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaMemcpyAsync(d_docids.p, docids, size_t(ndocs) * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_doff.p, doc_offsets, (size_t(ndocs) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        if (ntok) {
                CK(cudaMemcpyAsync(d_tok.p, tokens, ntok * 4, cudaMemcpyHostToDevice, c->stream));
                if (positions)
                        CK(cudaMemcpyAsync(d_pos.p, positions, ntok * 4, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaMemsetAsync(d_err.p, 0xff, sizeof herr, c->stream));
        const uint64_t doc_active = low_bits_for(ndocs - 1u) | (low_bits_for(max_docid) << 32);
        const uint64_t key_active = low_bits_for(positions ? 16383u : maxlen) | (low_bits_for(ndocs - 1u) << 14) | (low_bits_for(nterms - 1u) << 40);
        const auto     doc_passes = plan_radix_passes(doc_active), key_passes = plan_radix_passes(key_active);
        CK(cudaEventRecord(X.ev[0], c->stream));
        CK(launch_index_doc_keys(d_docids.as<uint32_t>(), ndocs, d_ka.as<unsigned long long>(), c->stream));
        unsigned long long *sorted{nullptr};
        if (const int r = index_radix_sort(c, d_ka, d_kb, ndocs, doc_passes, d_counts, d_part, d_offs, &sorted))
                return r;
        CK(launch_index_doc_ranks(sorted, ndocs, d_rank.as<uint32_t>(), d_docid_of.as<uint32_t>(), d_err.as<unsigned long long>(), c->stream));
        // ---- tokens: keys, the sort
        IndexParams P{};
        P.doc_off   = d_doff.as<unsigned long long>();
        P.tokens    = d_tok.as<uint32_t>();
        P.positions = positions ? d_pos.as<uint32_t>() : nullptr;
        P.plens     = with_payloads ? d_pl.as<uint8_t>() : nullptr;
        P.payloads  = with_payloads ? d_pv.as<unsigned long long>() : nullptr;
        P.ords      = with_payloads ? d_va.as<uint32_t>() : nullptr;
        P.ndocs     = ndocs;
        P.nterms    = nterms;
        P.ntokens   = ntok;
        P.rank_of   = d_rank.as<uint32_t>();
        P.docid_of  = d_docid_of.as<uint32_t>();
        P.keys      = d_ka.as<unsigned long long>();
        P.errors    = d_err.as<unsigned long long>();
        CK(launch_index_keys(P, c->stream));
        uint32_t *sorted_ords{nullptr};
        if (const int r = index_radix_sort(c, d_ka, d_kb, ntok, key_passes, d_counts, d_part, d_offs, &sorted, with_payloads ? &d_va : nullptr,
                                           with_payloads ? &d_vb : nullptr, &sorted_ords))
                return r;
        CK(cudaEventRecord(X.ev[1], c->stream));
        // ---- postings: flags and their scans
        CKM(d_pflag.ensure(std::max<uint64_t>(1, ntok) * 4));
        CKM(d_tflag.ensure(std::max<uint64_t>(1, ntok) * 4));
        CKM(d_pscan.ensure((ntok + 1) * 8));
        CKM(d_tscan.ensure((ntok + 1) * 8));
        CKM(d_part.ensure((ntok / 4096 + 4) * 8));
        CK(launch_post_flags(sorted, ntok, d_pflag.as<uint32_t>(), d_tflag.as<uint32_t>(), c->stream));
        CK(launch_enc_scan(d_pflag.as<uint32_t>(), ntok, d_part.as<unsigned long long>(), d_pscan.as<unsigned long long>(), c->stream));
        CK(launch_enc_scan(d_tflag.as<uint32_t>(), ntok, d_part.as<unsigned long long>(), d_tscan.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(X.ev[2], c->stream));
        uint64_t nposts{0}, npresent{0};
        CK(cudaMemcpyAsync(&nposts, d_pscan.as<unsigned long long>() + ntok, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&npresent, d_tscan.as<unsigned long long>() + ntok, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(herr, d_err.p, sizeof herr, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (herr[IDX_ERR_DOC0] != ~0ull)
                return fail(c, TRN_ERR_ARG, who(uint32_t(herr[IDX_ERR_DOC0])) + "docID 0 is not a document");
        if (herr[IDX_ERR_DUP] != ~0ull)
                return fail(c, TRN_ERR_ARG, who(uint32_t(herr[IDX_ERR_DUP])) + "the docID is given twice (Already committed document, indexer.cpp:219-222)");
        if (herr[IDX_ERR_TOKEN] != ~0ull) {
                const uint64_t i = herr[IDX_ERR_TOKEN];
                return fail(c, TRN_ERR_ARG, who(doc_of_token(i)) + "token " + std::to_string(i - doc_offsets[doc_of_token(i)]) + " is term " + std::to_string(tokens[i]) +
                                                ", not below nterms = " + std::to_string(nterms));
        }
        if (herr[IDX_ERR_POS] != ~0ull) {
                const uint64_t i = herr[IDX_ERR_POS];
                return fail(c, TRN_ERR_ARG, who(doc_of_token(i)) + "token " + std::to_string(i - doc_offsets[doc_of_token(i)]) + " has position " +
                                                std::to_string(positions ? positions[i] : 0u) + ": positions must be below 16384 (Limits::MaxPosition)");
        }
        if (herr[IDX_ERR_PAYLEN] != ~0ull) {
                const uint64_t i = herr[IDX_ERR_PAYLEN];
                return fail(c, TRN_ERR_ARG, who(doc_of_token(i)) + "token " + std::to_string(i - doc_offsets[doc_of_token(i)]) + " has a payload of " +
                                                std::to_string(payload_lens[i]) + " bytes: at most 8 (indexer.cpp:26)");
        }
        if (herr[IDX_ERR_POS0] != ~0ull) {
                const uint64_t i = herr[IDX_ERR_POS0];
                return fail(c, TRN_ERR_UNSUPPORTED, who(doc_of_token(i)) + "token " + std::to_string(i - doc_offsets[doc_of_token(i)]) +
                                                        " has position 0 and no payload: hits without a position are not indexed");
        }
        // ---- postings: docids, freqs, positions, term_begin in the layout the encode kernels read
        CKM(d_pbegin.ensure((nposts + 1) * 8));
        CKM(d_tb.ensure((npresent + 1) * 8));
        CKM(d_order.ensure(std::max<uint64_t>(1, npresent) * 4));
        CKM(d_odoc.ensure(std::max<uint64_t>(1, nposts) * 4));
        CKM(d_ofreq.ensure(std::max<uint64_t>(1, nposts) * 4));
        CKM(d_opos.ensure(std::max<uint64_t>(1, ntok) * 4));
        if (nterms > 65535u) {
                CKM(d_docterms.ensure(size_t(ndocs) * 4));
                CK(cudaMemsetAsync(d_docterms.p, 0, size_t(ndocs) * 4, c->stream));
        }
        P.post_flag     = d_pflag.as<uint32_t>();
        P.term_flag     = d_tflag.as<uint32_t>();
        P.post_scan     = d_pscan.as<unsigned long long>();
        P.term_scan     = d_tscan.as<unsigned long long>();
        P.post_begin    = d_pbegin.as<unsigned long long>();
        P.term_begin    = d_tb.as<unsigned long long>();
        P.term_order    = d_order.as<uint32_t>();
        P.out_docids    = d_odoc.as<uint32_t>();
        P.out_freqs     = d_ofreq.as<uint32_t>();
        P.out_positions = d_opos.as<uint32_t>();
        P.doc_terms     = nterms > 65535u ? d_docterms.as<uint32_t>() : nullptr;
        if (with_payloads) {
                CKM(d_opl.ensure(ntok));
                CKM(d_opv.ensure(ntok * 8));
                P.out_plens    = d_opl.as<uint8_t>();
                P.out_payloads = d_opv.as<unsigned long long>();
        }
        CK(cudaEventRecord(X.ev[3], c->stream));
        CK(launch_post_write(P, sorted, sorted_ords, c->stream));
        CK(launch_post_freqs(P, nposts, c->stream));
        CK(cudaEventRecord(X.ev[4], c->stream));
        std::vector<uint64_t> h_tb(npresent + 1);
        std::vector<uint32_t> h_order(npresent);
        CK(cudaMemcpyAsync(h_tb.data(), d_tb.p, (npresent + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        if (npresent)
                CK(cudaMemcpyAsync(h_order.data(), d_order.p, npresent * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(herr, d_err.p, sizeof herr, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (herr[IDX_ERR_FREQ] != ~0ull) {
                const uint64_t p = herr[IDX_ERR_FREQ];
                uint32_t       doc{0};
                CK(cudaMemcpy(&doc, d_odoc.as<uint32_t>() + p, 4, cudaMemcpyDeviceToHost));
                const size_t j = size_t(std::upper_bound(h_tb.begin(), h_tb.end(), p) - h_tb.begin()) - 1;
                return fail(c, TRN_ERR_ARG, "trn_index_documents: docID " + std::to_string(doc) + " holds term " + std::to_string(index_term_at(h_order[j], nterms)) +
                                                " more than 65535 times (a uint16_t count, indexer.cpp:102-103)");
        }
        if (herr[IDX_ERR_DOCTERMS] != ~0ull) {
                uint32_t doc{0};
                CK(cudaMemcpy(&doc, d_docid_of.as<uint32_t>() + herr[IDX_ERR_DOCTERMS], 4, cudaMemcpyDeviceToHost));
                return fail(c, TRN_ERR_ARG, "trn_index_documents: docID " + std::to_string(doc) + " holds more than 65535 distinct terms (a uint16_t count, indexer.cpp:49,111)");
        }
        if (herr[IDX_ERR_PAYDUP] != ~0ull) {
                unsigned long long k{0};
                uint32_t           doc{0};
                CK(cudaMemcpy(&k, sorted + herr[IDX_ERR_PAYDUP], 8, cudaMemcpyDeviceToHost));
                CK(cudaMemcpy(&doc, d_docid_of.as<uint32_t>() + ((k >> 14) & 0x3ffffffu), 4, cudaMemcpyDeviceToHost));
                return fail(c, TRN_ERR_UNSUPPORTED, "trn_index_documents: docID " + std::to_string(doc) + " holds term " + std::to_string(index_term_at(uint32_t(k >> 40), nterms)) +
                                                        " twice at position " + std::to_string(k & 16383u) +
                                                        " with different payloads: the reference leaves their order undefined (indexer.cpp:55-57)");
        }
        float sort_ms{0}, a_ms{0}, b_ms{0}, enc_ms{0};
        CK(cudaEventElapsedTime(&sort_ms, X.ev[0], X.ev[1]));
        CK(cudaEventElapsedTime(&a_ms, X.ev[1], X.ev[2]));
        CK(cudaEventElapsedTime(&b_ms, X.ev[3], X.ev[4]));
        for (DevBuf *b : {&d_docids, &d_doff, &d_tok, &d_pos, &d_ka, &d_kb, &d_rank, &d_docid_of, &d_counts, &d_part, &d_offs, &d_pflag, &d_tflag, &d_pscan, &d_tscan,
                          &d_pbegin, &d_order, &d_docterms, &d_pl, &d_pv, &d_va, &d_vb})
                b->release();
        // ---- encode the device-resident postings: terms in index order, the reference's geometry, a fresh session
        std::vector<uint8_t>  index, hits;
        std::vector<trn_term> terms(nterms, trn_term{0, 0, 0});
        std::vector<uint64_t> chunk, toff;
        uint64_t              index_bytes{0}, hits_bytes{0};
        if (npresent) {
                DevPostings DP{h_tb.data(), uint32_t(npresent), d_tb.as<unsigned long long>(), d_odoc.as<uint32_t>(), d_ofreq.as<uint32_t>(), d_opos.as<uint32_t>()};
                if (with_payloads) {
                        DP.plens    = d_opl.as<uint8_t>();
                        DP.payloads = d_opv.as<unsigned long long>();
                }
                int r;
                if (codec == TRN_CODEC_GOOGLE) {
                        uint64_t nblocks{0};
                        r = encode_google_device(c, DP, 32, 8, 0, true, ~0ull, &index_bytes, d_out, chunk, toff, &nblocks, &enc_ms);
                } else
                        r = encode_lucene_device(c, DP, true, ~0ull, &index_bytes, true, ~0ull, &hits_bytes, d_out, d_hout, toff, &enc_ms);
                if (r == TRN_ERR_CUDA && c->err.find("out of memory") != std::string::npos)
                        return fail(c, TRN_ERR_CAPACITY, "trn_index_documents: working memory cannot be allocated on the device; split the batch");
                if (r)
                        return r;
                try {
                        index.resize(index_bytes);
                        hits.resize(hits_bytes);
                } catch (const std::bad_alloc &) {
                        return fail(c, TRN_ERR_CAPACITY, "trn_index_documents: the result cannot be allocated on the host");
                }
                CK(cudaMemcpyAsync(index.data(), d_out.p, index_bytes, cudaMemcpyDeviceToHost, c->stream));
                if (hits_bytes)
                        CK(cudaMemcpyAsync(hits.data(), d_hout.p, hits_bytes, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                for (size_t j = 0; j < npresent; ++j) {
                        trn_term &t = terms[index_term_at(h_order[j], nterms)];
                        t.documents = uint32_t(h_tb[j + 1] - h_tb[j]);
                        t.chunk_off = uint32_t(toff[j]);
                        t.chunk_len = uint32_t(toff[j + 1] - toff[j]);
                }
        }
        X.index.swap(index);
        X.hits.swap(hits);
        X.terms.swap(terms);
        *out                = trn_indexed{};
        out->index          = X.index.data();
        out->index_bytes    = X.index.size();
        out->hits           = X.hits.data();
        out->hits_bytes     = X.hits.size();
        out->terms          = X.terms.data();
        out->nterms         = nterms;
        out->docs_cnt       = docs_cnt;
        out->total_terms    = uint32_t(npresent);
        out->sum_terms_docs = nposts;
        out->sum_term_hits  = ntok;
        out->max_docid      = max_docid;
        out->sort_passes    = uint32_t(doc_passes.size() + key_passes.size());
        out->sort_ms        = sort_ms;
        out->postings_ms    = a_ms + b_ms;
        out->encode_ms      = enc_ms;
        out->total_ms       = float(now_ms() - t_begin);
        return TRN_OK;
}

extern "C" int trn_index_documents(trn_ctx *c, int codec, const uint32_t *docids, const uint64_t *doc_offsets, const uint32_t *tokens, const uint32_t *positions,
                                   uint32_t ndocs, uint32_t nterms, trn_indexed *out) {
        return trn_index_documents_payloads(c, codec, docids, doc_offsets, tokens, positions, nullptr, nullptr, ndocs, nterms, out);
}

// =================================================================================================== decode probe
extern "C" int trn_decode_terms(trn_ctx *c, const uint32_t *term_ids, uint32_t nterms, int materialise, uint32_t *docids, uint32_t *freqs, uint64_t *sums,
                                float *device_ms) {
        if (!c)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (!term_ids || !nterms || (materialise && (!docids || !freqs)))
                return fail(c, TRN_ERR_ARG, "trn_decode_terms: bad arguments");
        CK(cudaSetDevice(c->device));
        std::vector<uint32_t> unit_base(nterms);
        std::vector<uint64_t> out_base(nterms + 1), host_base(nterms + 1);
        uint64_t              units{0}, posts{0}, padded{0};
        for (uint32_t i = 0; i < nterms; ++i) {
                if (term_ids[i] >= c->nterms)
                        return fail(c, TRN_ERR_ARG, "term id out of range");
                const auto &t = c->h_terms[term_ids[i]];
                unit_base[i]  = uint32_t(units);
                out_base[i]   = padded; // device rows start on a 128-entry boundary (16-byte vector stores)
                host_base[i]  = posts;
                units += (t.nblocks + 31) / 32;
                posts += t.documents;
                padded += (uint64_t(t.documents) + 127) / 128 * 128;
                if (units >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, "too many decode units");
        }
        out_base[nterms]  = padded;
        host_base[nterms] = posts;
        { // unit descriptors of the streaming kernels (decode_stream.cuh)
                std::vector<DecUnit> du(units);
                const uint32_t       bd = c->block_docs;
                for (uint32_t i = 0; i < nterms; ++i) {
                        const auto &t = c->h_terms[term_ids[i]];
                        for (uint32_t g0 = 0, u = unit_base[i]; g0 < t.nblocks; g0 += 32, ++u) {
                                DecUnit &D    = du[u];
                                D.first_entry = t.dir_begin + g0;
                                D.cnt         = std::min(32u, t.nblocks - g0);
                                D.term_start  = g0 == 0;
                                const uint32_t lastN = t.documents - bd * (t.nblocks - 1u); // documents of the term's last block
                                D.last_n      = (g0 + D.cnt == t.nblocks && (c->pc.codec == TRN_CODEC_GOOGLE ? true : lastN != bd)) ? lastN : 0u;
                                if (c->pc.codec == TRN_CODEC_LUCENE && (t.documents & 127u) == 0u)
                                        D.last_n = 0;
                                D.ti   = i;
                                D.g0   = g0;
                                D.pad0 = D.pad1 = 0;
                        }
                }
                CK(c->d_dec_units.ensure(std::max<size_t>(32, du.size() * sizeof(DecUnit))));
                if (!du.empty())
                        CK(cudaMemcpyAsync(c->d_dec_units.p, du.data(), du.size() * sizeof(DecUnit), cudaMemcpyHostToDevice, c->stream));
                CK(cudaStreamSynchronize(c->stream)); // `du` leaves scope
        }
        CK(c->d_dec_c.ensure((nterms + 1) * 8));
        CK(c->d_dec_sums.ensure(size_t(nterms) * 16));
        if (materialise) {
                CK(c->d_dec_docids.ensure(std::max<size_t>(16, padded * 4)));
                CK(c->d_dec_freqs.ensure(std::max<size_t>(16, padded * 4)));
        }
        CK(cudaMemcpyAsync(c->d_dec_c.p, out_base.data(), (nterms + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemsetAsync(c->d_dec_sums.p, 0, size_t(nterms) * 16, c->stream));
        CK(cudaEventRecord(c->ev0, c->stream));
        if (units)
                CK(launch_decode_stream(dev_index(c), c->d_dec_units.as<DecUnit>(), c->d_dec_c.as<uint64_t>(), uint32_t(units),
                                        materialise ? c->d_dec_docids.as<uint32_t>() : nullptr, materialise ? c->d_dec_freqs.as<uint32_t>() : nullptr,
                                        c->d_dec_sums.as<unsigned long long>(), c->num_sms, c->stream));
        CK(cudaEventRecord(c->ev1, c->stream));
        if (materialise && posts) {
                for (uint32_t i = 0; i < nterms; ++i) {
                        const uint64_t n = host_base[i + 1] - host_base[i];
                        if (!n)
                                continue;
                        CK(cudaMemcpyAsync(docids + host_base[i], c->d_dec_docids.as<uint32_t>() + out_base[i], n * 4, cudaMemcpyDeviceToHost, c->stream));
                        CK(cudaMemcpyAsync(freqs + host_base[i], c->d_dec_freqs.as<uint32_t>() + out_base[i], n * 4, cudaMemcpyDeviceToHost, c->stream));
                }
        }
        if (sums)
                CK(cudaMemcpyAsync(sums, c->d_dec_sums.p, size_t(nterms) * 16, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (device_ms) {
                float ms{0};
                CK(cudaEventElapsedTime(&ms, c->ev0, c->ev1));
                *device_ms = ms;
        }
        return TRN_OK;
}

// =================================================================================================== query-token intersections
// Two device passes with the epoch planner between them (intersect.cuh, isectplan.h; DESIGN.md §4).  Three host synchronisations: the
// distinct-mask counts after pass A (to refuse a request over the limit and to lay out the dense copy), that copy, and the counts.
extern "C" int trn_intersect(trn_ctx *c, const trn_isect_req *reqs, uint32_t n, trn_intersections *out) {
        if (!c)
                return TRN_ERR_ARG;
        if (!out || (n && !reqs))
                return fail(c, TRN_ERR_ARG, "trn_intersect: bad arguments");
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (c->pc.codec == TRN_CODEC_GOOGLE && c->block_docs != 32)
                return fail(c, TRN_ERR_UNSUPPORTED, "the uploaded index was built with a block size other than the reference format's (decode sweep only)");
        CK(cudaSetDevice(c->device));
        std::memset(out, 0, sizeof(*out));
        const double t0 = now_ms();
        auto &       B  = c->it;
        if (!B.ev[0])
                for (Event &e : B.ev)
                        CK(cudaEventCreate(&e.h));

        // ---- the requests: known tokens (deduplicated per group), tile geometry, mask tables
        std::vector<IsectReq> rq(n);
        std::vector<uint2>    tok;
        uint64_t              items = 0, slots = 0, postings = 0;
        for (uint32_t i = 0; i < n; ++i) {
                const trn_isect_req &q   = reqs[i];
                const std::string    who = "trn_intersect: request " + std::to_string(i) + ": ";
                if (q.ngroups > 64)
                        return fail(c, TRN_ERR_ARG, who + std::to_string(q.ngroups) + " token groups (at most 64: one bit of a 64-bit mask each)");
                if (q.stopwords_mask)
                        return fail(c, TRN_ERR_UNSUPPORTED, who + "a non-zero stopwords mask (the reference tests it against iterator slots, whose order is not reproducible)");
                if (q.ngroups && !q.group_offsets)
                        return fail(c, TRN_ERR_ARG, who + "null group_offsets");
                IsectReq &R = rq[i];
                std::memset(&R, 0, sizeof(R));
                R.tok_begin = uint32_t(tok.size());
                R.ngroups   = q.ngroups;
                R.shift     = isect_tile_shift(q.ngroups);
                bool     unknown{false};
                uint64_t orig{0}, docs{0};
                uint32_t lo{0xffffffffu}, hi{0};
                for (uint32_t g = 0; g < q.ngroups; ++g) {
                        const uint32_t a = q.group_offsets[g], b = q.group_offsets[g + 1];
                        if (b < a || (b > a && !q.terms))
                                return fail(c, TRN_ERR_ARG, who + "group_offsets must not decrease, and terms must be given");
                        std::vector<uint32_t> ts(q.terms + a, q.terms + b);
                        std::sort(ts.begin(), ts.end());
                        ts.erase(std::unique(ts.begin(), ts.end()), ts.end());
                        for (const uint32_t t : ts) {
                                if (t != TRN_EMPTY_TERM && t >= c->nterms)
                                        return fail(c, TRN_ERR_ARG, who + "term id " + std::to_string(t) + " out of range");
                                if (t == TRN_EMPTY_TERM || !c->h_terms[t].documents) {
                                        unknown = true;
                                        continue;
                                }
                                const DevTerm &T = c->h_terms[t];
                                tok.push_back(make_uint2(t, g));
                                orig |= 1ull << g;
                                lo = std::min(lo, T.first_doc);
                                hi = std::max(hi, T.last_doc);
                                docs += T.documents;
                        }
                }
                R.ntok = uint32_t(tok.size()) - R.tok_begin;
                if (R.ntok > 512)
                        return fail(c, TRN_ERR_ARG, who + std::to_string(R.ntok) + " known tokens (at most 512, the reference's iterator slots; a token in two groups takes two)");
                postings += docs;
                R.orig_mask  = unknown ? 0ull : orig;
                R.item_base  = uint32_t(items);
                R.table_base = slots;
                if (!R.ntok)
                        continue; // nothing to intersect: an empty result
                R.tile_lo = lo >> R.shift;
                R.ntiles  = (hi >> R.shift) - R.tile_lo + 1u;
                items += R.ntiles;
                uint64_t bound = std::min<uint64_t>(c->isect_max_masks, docs); // distinct masks can be no more than the documents ...
                if (q.ngroups < 64)
                        bound = std::min<uint64_t>(bound, (1ull << q.ngroups) - 1u); // ... or the non-empty masks
                uint64_t s = 64;
                while (s < 2u * (bound + 1u)) // one more than the limit must fit, to be seen
                        s <<= 1;
                R.slots = s;
                slots += s;
        }
        if (items >= (1ull << 31))
                return fail(c, TRN_ERR_CAPACITY, "trn_intersect: the batch covers " + std::to_string(items) + " docID tiles; split it");

        auto upload = [&](DevBuf &b, const void *src, size_t bytes) -> cudaError_t {
                if (const cudaError_t e = b.ensure(std::max<size_t>(16, bytes)); e != cudaSuccess)
                        return e;
                return bytes ? cudaMemcpyAsync(b.p, src, bytes, cudaMemcpyHostToDevice, c->stream) : cudaSuccess;
        };
        const bool  luc = c->pc.codec == TRN_CODEC_LUCENE;
        IsectParams P;
        std::memset(&P, 0, sizeof(P));
        P.ix          = dev_index(c);
        P.nreq        = n;
        P.total_items = uint32_t(items);
        P.max_masks   = c->isect_max_masks;
        // small: ticket, error, ndist[n], compact cursors[n]
        CK(B.d_small.ensure((2 + 2 * size_t(n)) * 4));
        CK(cudaMemsetAsync(B.d_small.p, 0, (2 + 2 * size_t(n)) * 4, c->stream));
        P.ticket = B.d_small.as<uint32_t>();
        P.error  = P.ticket + 1;
        P.ndist  = P.ticket + 2;
        CK(upload(B.d_tok, tok.data(), tok.size() * sizeof(uint2)));
        P.tok = B.d_tok.as<uint2>();
        CK(B.d_keys.ensure(std::max<size_t>(16, slots * 8)));
        CK(B.d_first.ensure(std::max<size_t>(16, slots * 4)));
        CK(B.d_tile_last.ensure(std::max<size_t>(16, items * 8)));
        CK(cudaMemsetAsync(B.d_keys.p, 0, slots * 8, c->stream));
        CK(cudaMemsetAsync(B.d_first.p, 0xff, slots * 4, c->stream));
        P.keys      = B.d_keys.as<unsigned long long>();
        P.first     = B.d_first.as<uint32_t>();
        P.tile_last = B.d_tile_last.as<unsigned long long>();

        // ---- pass A: the distinct masks of every request with their first docIDs, and every tile's last considered mask
        CK(upload(B.d_reqs, rq.data(), rq.size() * sizeof(IsectReq)));
        P.reqs = B.d_reqs.as<IsectReq>();
        CK(cudaEventRecord(B.ev[0], c->stream));
        if (items)
                CK(launch_isect(P, luc, false, c->num_sms, c->stream));
        CK(cudaEventRecord(B.ev[1], c->stream));
        std::vector<uint32_t> small(2 + size_t(n));
        CK(cudaMemcpyAsync(small.data(), B.d_small.p, small.size() * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        for (uint32_t i = 0; i < n; ++i)
                if (small[2 + i] > c->isect_max_masks)
                        return fail(c, TRN_ERR_CAPACITY, "trn_intersect: request " + std::to_string(i) + " has more than " + std::to_string(c->isect_max_masks) +
                                                              " distinct token masks; TRN_ISECT_MAX_MASKS may only lower that limit");
        if (small[1])
                return fail(c, TRN_ERR_CAPACITY, "trn_intersect: a mask table overflowed (internal bound violated)");
        float masksMs{0};
        (void)cudaEventElapsedTime(&masksMs, B.ev[0], B.ev[1]);

        // ---- the distinct masks, densely, to the host
        std::vector<uint64_t> base(size_t(n) + 1, 0);
        for (uint32_t i = 0; i < n; ++i)
                base[i + 1] = base[i] + small[2 + i];
        const uint64_t        D = base[n];
        std::vector<uint64_t> hmask(D);
        std::vector<uint32_t> hfirst(D);
        if (D) {
                CK(upload(B.d_base, base.data(), base.size() * 8));
                CK(B.d_cmask.ensure(D * 8));
                CK(B.d_cfirst.ensure(D * 4));
                CK(launch_isect_compact(P, slots, B.d_base.as<uint64_t>(), P.ndist + n, B.d_cmask.as<unsigned long long>(), B.d_cfirst.as<uint32_t>(), c->num_sms,
                                        c->stream));
                CK(cudaMemcpyAsync(hmask.data(), B.d_cmask.p, D * 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(hfirst.data(), B.d_cfirst.p, D * 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
        }

        // ---- host step: every request's epochs and their arrays
        const double          th = now_ms();
        std::vector<uint32_t> estart, eoff;
        std::vector<uint64_t> smask, fmask;
        std::vector<int32_t>  sslot;
        std::vector<uint64_t> fbase(size_t(n) + 1, 0);
        for (uint32_t i = 0; i < n; ++i) {
                IsectPlan   pl;
                std::string err;
                if (isect_plan(hmask.data() + base[i], hfirst.data() + base[i], small[2 + i], c->isect_max_masks, pl, err))
                        return fail(c, TRN_ERR_CAPACITY, "trn_intersect: request " + std::to_string(i) + ": " + err);
                IsectReq &R   = rq[i];
                R.epoch_begin = uint32_t(estart.size());
                R.nepochs     = uint32_t(pl.epoch_start.size());
                const uint32_t sb = uint32_t(smask.size()), fb = uint32_t(fmask.size());
                estart.insert(estart.end(), pl.epoch_start.begin(), pl.epoch_start.end());
                for (size_t e = 0; e < pl.epoch_start.size(); ++e)
                        eoff.push_back(sb + pl.epoch_off[e]);
                smask.insert(smask.end(), pl.snap_mask.begin(), pl.snap_mask.end());
                for (const int32_t s : pl.snap_slot)
                        sslot.push_back(s < 0 ? -1 : int32_t(fb) + s);
                fmask.insert(fmask.end(), pl.final_mask.begin(), pl.final_mask.end());
                fbase[i + 1] = fmask.size();
        }
        eoff.push_back(uint32_t(smask.size()));
        const float planMs = float(now_ms() - th);

        // ---- pass B: every considered document's contribution to its target's final count
        std::vector<uint32_t> counts(fmask.size());
        float                 countMs{0};
        if (D) {
                CK(upload(B.d_reqs, rq.data(), rq.size() * sizeof(IsectReq)));
                CK(upload(B.d_estart, estart.data(), estart.size() * 4));
                CK(upload(B.d_eoff, eoff.data(), eoff.size() * 4));
                CK(upload(B.d_smask, smask.data(), smask.size() * 8));
                CK(upload(B.d_sslot, sslot.data(), sslot.size() * 4));
                CK(B.d_counts.ensure(std::max<size_t>(16, counts.size() * 4)));
                CK(cudaMemsetAsync(B.d_counts.p, 0, counts.size() * 4, c->stream));
                CK(B.d_carry.ensure(std::max<size_t>(16, items * 8)));
                CK(cudaMemsetAsync(P.ticket, 0, 4, c->stream));
                P.carry       = B.d_carry.as<unsigned long long>();
                P.epoch_start = B.d_estart.as<uint32_t>();
                P.epoch_off   = B.d_eoff.as<uint32_t>();
                P.snap_mask   = B.d_smask.as<unsigned long long>();
                P.snap_slot   = B.d_sslot.as<int32_t>();
                P.counts      = B.d_counts.as<uint32_t>();
                CK(cudaEventRecord(B.ev[2], c->stream));
                CK(launch_isect_carry(P, B.d_carry.as<unsigned long long>(), c->stream));
                CK(launch_isect(P, luc, true, c->num_sms, c->stream));
                CK(cudaEventRecord(B.ev[3], c->stream));
                CK(cudaMemcpyAsync(counts.data(), B.d_counts.p, counts.size() * 4, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaMemcpyAsync(small.data(), B.d_small.p, 8, cudaMemcpyDeviceToHost, c->stream));
                CK(cudaStreamSynchronize(c->stream));
                if (small[1])
                        return fail(c, TRN_ERR_STATE, "trn_intersect: a considered document found no entry in its epoch's array (internal error)");
                (void)cudaEventElapsedTime(&countMs, B.ev[2], B.ev[3]);
        }

        // ---- the result, in finalize()'s order with ties broken by mask
        B.offsets.assign(size_t(n) + 1, 0);
        B.masks.clear();
        B.counts.clear();
        for (uint32_t i = 0; i < n; ++i) {
                std::vector<uint32_t> ord(fbase[i + 1] - fbase[i]);
                std::iota(ord.begin(), ord.end(), uint32_t(fbase[i]));
                std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return isect_result_less(fmask[a], counts[a], fmask[b], counts[b]); });
                for (const uint32_t j : ord) {
                        B.masks.push_back(fmask[j]);
                        B.counts.push_back(counts[j]);
                }
                B.offsets[i + 1] = B.masks.size();
        }
        out->n        = n;
        out->total    = B.masks.size();
        out->offsets  = B.offsets.data();
        out->masks    = B.masks.data();
        out->counts   = B.counts.data();
        out->postings = postings;
        out->distinct = D;
        out->masks_ms = masksMs;
        out->plan_ms  = planMs;
        out->count_ms = countMs;
        out->total_ms = float(now_ms() - t0);
        return TRN_OK;
}

extern "C" int trn_debug_intersect_plan(const uint64_t *masks, const uint32_t *firsts, uint32_t n, uint32_t max_masks, uint32_t *epoch_start, uint32_t *epoch_off,
                                        uint64_t *snap_mask, int32_t *snap_slot, uint64_t cap, uint32_t *nepochs, uint64_t *nentries, uint64_t *final_mask,
                                        uint32_t *nfinal, char *err, size_t errcap) {
        auto say = [&](const std::string &m) {
                if (err && errcap)
                        snprintf(err, errcap, "%s", m.c_str());
        };
        if ((n && (!masks || !firsts)) || !epoch_start || !epoch_off || !nepochs || !nentries || !final_mask || !nfinal || (cap && (!snap_mask || !snap_slot))) {
                say("trn_debug_intersect_plan: bad arguments");
                return TRN_ERR_ARG;
        }
        IsectPlan   pl;
        std::string e;
        if (isect_plan(masks, firsts, n, max_masks ? max_masks : kIsectMaxMasks, pl, e)) {
                say(e);
                return TRN_ERR_CAPACITY;
        }
        *nepochs  = uint32_t(pl.epoch_start.size());
        *nentries = pl.snap_mask.size();
        *nfinal   = uint32_t(pl.final_mask.size());
        if (pl.snap_mask.size() > cap) {
                say("trn_debug_intersect_plan: " + std::to_string(pl.snap_mask.size()) + " entries do not fit");
                return TRN_ERR_CAPACITY;
        }
        std::copy(pl.epoch_start.begin(), pl.epoch_start.end(), epoch_start);
        std::copy(pl.epoch_off.begin(), pl.epoch_off.end(), epoch_off);
        std::copy(pl.snap_mask.begin(), pl.snap_mask.end(), snap_mask);
        std::copy(pl.snap_slot.begin(), pl.snap_slot.end(), snap_slot);
        std::copy(pl.final_mask.begin(), pl.final_mask.end(), final_mask);
        return TRN_OK;
}

// =================================================================================================== percolator
// Registration plans on the host (percplan.h) and uploads the registry; trn_percolate runs the count pass, scans the counts, sizes the
// result once from them and runs the write pass (percolate.cuh; DESIGN.md §4).  Two host synchronisations: the offsets after the scan, the
// result.
extern "C" int trn_percolator_register(trn_ctx *c, const trn_query *queries, uint32_t nq, uint32_t nterms, const uint32_t *term_cost, trn_percolator_info *out) {
        if (!c)
                return TRN_ERR_ARG;
        if (nq && !queries)
                return fail(c, TRN_ERR_ARG, "trn_percolator_register: bad arguments");
        CK(cudaSetDevice(c->device));
        PercPlan    P;
        std::string err;
        if (const int rc = perc_plan(queries, nq, nterms, term_cost, P, err))
                return fail(c, rc, "trn_percolator_register: " + err);
        if (nq > c->perc_max_ids || P.csr.size() >= c->perc_max_entries)
                return fail(c, TRN_ERR_CAPACITY, "trn_percolator_register: " + std::to_string(nq) + " queries with " + std::to_string(P.csr.size()) +
                                                     " anchor entries exceed the registry's limits");
        auto &B = c->pq;
        B.have  = false;
        uint64_t bytes{0};
        auto     upload = [&](DevBuf &b, const void *src, size_t n) -> cudaError_t {
                bytes += n;
                if (const cudaError_t e = b.ensure(std::max<size_t>(16, n)); e != cudaSuccess)
                        return e;
                return n ? cudaMemcpyAsync(b.p, src, n, cudaMemcpyHostToDevice, c->stream) : cudaSuccess;
        };
        CK(upload(B.d_queries, P.queries.data(), P.queries.size() * sizeof(PercQuery)));
        CK(upload(B.d_ops, P.ops.data(), P.ops.size() * sizeof(PercOp)));
        CK(upload(B.d_pterms, P.phrase_terms.data(), P.phrase_terms.size() * 4));
        CK(upload(B.d_covers, P.covers.data(), P.covers.size() * 4));
        CK(upload(B.d_csr_off, P.csr_off.data(), P.csr_off.size() * 4));
        CK(upload(B.d_csr, P.csr.data(), P.csr.size() * sizeof(PercEntry)));
        CK(upload(B.d_unanch, P.unanchored.data(), P.unanchored.size() * 4));
        CK(cudaStreamSynchronize(c->stream));
        B.next_id     = nq;
        B.nterms      = nterms;
        B.nunanchored = uint32_t(P.unanchored.size());
        B.sizes.resize(nq);
        for (uint32_t q = 0; q < nq; ++q)
                B.sizes[q] = {P.queries[q].nops, P.npt[q], P.queries[q].ncover, P.status[q]};
        B.removed.assign((size_t(nq) + 31u) / 32u, 0u);
        B.term_cost.assign(term_cost, term_cost ? term_cost + nterms : term_cost);
        B.nlive       = nq;
        B.nnever      = P.never;
        B.nentries    = P.csr.size();
        B.ops_used    = P.ops.size();
        B.pt_used     = P.phrase_terms.size();
        B.cov_used    = P.covers.size();
        B.dead_words  = 0;
        B.info        = trn_percolator_info{nq, B.nunanchored, P.never, nq, P.csr.size(), bytes};
        B.have        = true;
        if (out)
                *out = B.info;
        return TRN_OK;
}

extern "C" int trn_percolate(trn_ctx *c, const uint64_t *doc_offsets, const uint32_t *tokens, uint32_t ndocs, trn_percolation *out) {
        if (!c)
                return TRN_ERR_ARG;
        if (!out || (ndocs && !doc_offsets))
                return fail(c, TRN_ERR_ARG, "trn_percolate: bad arguments");
        auto &B = c->pq;
        if (!B.have)
                return fail(c, TRN_ERR_STATE, "trn_percolate: no query set registered (trn_percolator_register)");
        CK(cudaSetDevice(c->device));
        std::memset(out, 0, sizeof(*out));
        const double t0 = now_ms();
        if (!B.ev[0])
                for (Event &e : B.ev)
                        CK(cudaEventCreate(&e.h));

        // ---- the documents: lengths, tokens, the short and the long launch
        const uint64_t base = ndocs ? doc_offsets[0] : 0, ntok = ndocs ? doc_offsets[ndocs] - base : 0;
        if (ntok && !tokens)
                return fail(c, TRN_ERR_ARG, "trn_percolate: bad arguments");
        std::vector<uint32_t> docs[2];
        uint32_t              max_len[2]{0, 0};
        std::vector<uint64_t> off(size_t(ndocs) + 1, 0);
        for (uint32_t d = 0; d < ndocs; ++d) {
                const std::string who = "trn_percolate: document " + std::to_string(d) + ": ";
                if (doc_offsets[d + 1] < doc_offsets[d] || doc_offsets[d + 1] - base > ntok)
                        return fail(c, TRN_ERR_ARG, who + "doc_offsets must not decrease");
                const uint64_t L = doc_offsets[d + 1] - doc_offsets[d];
                if (L > kPercMaxDocLen)
                        return fail(c, TRN_ERR_ARG, who + std::to_string(L) + " tokens (at most 16383: positions below Limits::MaxPosition)");
                for (uint64_t i = doc_offsets[d]; i < doc_offsets[d + 1]; ++i)
                        if (tokens[i] != kEmptyTerm && tokens[i] >= B.nterms)
                                return fail(c, TRN_ERR_ARG, who + "token id " + std::to_string(tokens[i]) + " outside the vocabulary (use TRN_EMPTY_TERM)");
                const int lg = L > kPercShortLen;
                docs[lg].push_back(d);
                max_len[lg] = std::max(max_len[lg], uint32_t(L));
                off[d + 1]  = doc_offsets[d + 1] - base;
        }
        auto upload = [&](DevBuf &b, const void *src, size_t n) -> cudaError_t {
                if (const cudaError_t e = b.ensure(std::max<size_t>(16, n)); e != cudaSuccess)
                        return e;
                return n ? cudaMemcpyAsync(b.p, src, n, cudaMemcpyHostToDevice, c->stream) : cudaSuccess;
        };
        CK(upload(B.d_doc_off, off.data(), off.size() * 8));
        CK(upload(B.d_tokens, tokens + base, ntok * 4));
        CK(B.d_docs.ensure(std::max<size_t>(16, size_t(ndocs) * 4)));
        CK(cudaMemcpyAsync(B.d_docs.p, docs[0].data(), docs[0].size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(B.d_docs.as<uint32_t>() + docs[0].size(), docs[1].data(), docs[1].size() * 4, cudaMemcpyHostToDevice, c->stream));
        CK(B.d_counts.ensure(std::max<size_t>(16, size_t(ndocs) * 4)));
        CK(B.d_small.ensure(16));
        CK(cudaMemsetAsync(B.d_small.p, 0, 8, c->stream));
        CK(B.d_part.ensure((size_t(ndocs) / 4096 + 2) * 8));
        CK(B.d_out_off.ensure((size_t(ndocs) + 1) * 8));

        PercParams P;
        std::memset(&P, 0, sizeof(P));
        P.queries      = B.d_queries.as<PercQuery>();
        P.ops          = B.d_ops.as<PercOp>();
        P.phrase_terms = B.d_pterms.as<uint32_t>();
        P.covers       = B.d_covers.as<uint32_t>();
        P.csr_off      = B.d_csr_off.as<uint32_t>();
        P.csr          = B.d_csr.as<PercEntry>();
        P.unanchored   = B.d_unanch.as<uint32_t>();
        P.nunanchored  = B.nunanchored;
        P.nterms       = B.nterms;
        P.doc_off      = B.d_doc_off.as<unsigned long long>();
        P.tokens       = B.d_tokens.as<uint32_t>();
        P.counts       = B.d_counts.as<uint32_t>();
        P.candidates   = B.d_small.as<unsigned long long>();
        auto launches  = [&](bool write) -> cudaError_t {
                for (int lg = 0; lg < 2; ++lg) {
                        PercParams L = P;
                        L.docs       = B.d_docs.as<uint32_t>() + (lg ? docs[0].size() : 0);
                        L.ndocs      = uint32_t(docs[lg].size());
                        L.max_len    = max_len[lg];
                        L.max_hash   = perc_hash_slots(max_len[lg]);
                        if (const cudaError_t e = launch_perc(L, write, c->num_sms, c->stream); e != cudaSuccess)
                                return e;
                }
                return cudaSuccess;
        };

        // ---- count pass and the scan of the counts
        CK(cudaEventRecord(B.ev[0], c->stream));
        CK(launches(false));
        CK(launch_enc_scan(P.counts, ndocs, B.d_part.as<unsigned long long>(), B.d_out_off.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(B.ev[1], c->stream));
        CK(B.h_offsets.ensure((size_t(ndocs) + 1) * 8));
        uint64_t cand{0};
        CK(cudaMemcpyAsync(B.h_offsets.p, B.d_out_off.p, (size_t(ndocs) + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&cand, B.d_small.p, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        const uint64_t *hoff  = B.h_offsets.as<uint64_t>();
        const uint64_t  total = hoff[ndocs];

        // ---- the result, sized once; a bitmap per document with more matches than shared memory sorts
        std::vector<uint32_t> slot(ndocs, 0);
        uint32_t              ndense{0};
        for (uint32_t d = 0; d < ndocs; ++d)
                if (hoff[d + 1] - hoff[d] > kPercSortCap)
                        slot[d] = ndense++;
        const uint32_t words = (B.next_id + 31u) / 32u;
        auto capacity = [&](cudaError_t e, const char *what) {
                (void)cudaGetLastError();
                return fail(c, e == cudaErrorMemoryAllocation ? TRN_ERR_CAPACITY : TRN_ERR_CUDA,
                            std::string("trn_percolate: ") + what + " (" + std::to_string(total) + " matches): " + cudaGetErrorString(e) + "; split the batch");
        };
        if (const cudaError_t e = B.d_out.ensure(std::max<size_t>(16, total * 4)); e != cudaSuccess)
                return capacity(e, "the matches cannot be staged on the device");
        if (const cudaError_t e = B.h_ids.ensure(std::max<size_t>(16, total * 4)); e != cudaSuccess)
                return capacity(e, "the pinned result cannot be allocated");
        if (ndense) {
                if (const cudaError_t e = B.d_bitmaps.ensure(size_t(ndense) * words * 4); e != cudaSuccess)
                        return capacity(e, "the bitmaps of the documents with many matches cannot be allocated");
                CK(cudaMemsetAsync(B.d_bitmaps.p, 0, size_t(ndense) * words * 4, c->stream));
        }
        CK(upload(B.d_dense_slot, slot.data(), slot.size() * 4));
        P.out_off      = B.d_out_off.as<unsigned long long>();
        P.out          = B.d_out.as<uint32_t>();
        P.bitmaps      = B.d_bitmaps.as<uint32_t>();
        P.dense_slot   = B.d_dense_slot.as<uint32_t>();
        P.bitmap_words = words;

        // ---- write pass
        CK(cudaEventRecord(B.ev[2], c->stream));
        CK(launches(true));
        CK(cudaEventRecord(B.ev[3], c->stream));
        CK(cudaMemcpyAsync(B.h_ids.p, B.d_out.p, total * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        float countMs{0}, writeMs{0};
        (void)cudaEventElapsedTime(&countMs, B.ev[0], B.ev[1]);
        (void)cudaEventElapsedTime(&writeMs, B.ev[2], B.ev[3]);
        out->ndocs      = ndocs;
        out->long_docs  = uint32_t(docs[1].size());
        out->dense_docs = ndense;
        out->total      = total;
        out->offsets    = hoff;
        out->queries    = B.h_ids.as<uint32_t>();
        out->candidates = cand;
        out->count_ms   = countMs;
        out->write_ms   = writeMs;
        out->total_ms   = float(now_ms() - t0);
        return TRN_OK;
}

// ---- trn_percolator_add / trn_percolator_remove (DESIGN.md §4): the added queries are planned on the host (perc_plan_queries on the slice)
// and their programs appended; the anchor index and the unanchored list are rebuilt on the device (percolate_update.cuh) into new buffers,
// and program storage that grows or is compacted goes to new buffers too.  They replace the old ones only once every step has succeeded, so
// a refused or failed call leaves the registry, and the last trn_percolate result, as they were.
#define CKPU(call)                                                                                                                                             \
        do {                                                                                                                                                   \
                cudaError_t e__ = (call);                                                                                                                      \
                if (e__ != cudaSuccess) {                                                                                                                      \
                        (void)cudaGetLastError();                                                                                                              \
                        return fail(c, e__ == cudaErrorMemoryAllocation ? TRN_ERR_CAPACITY : TRN_ERR_CUDA,                                                    \
                                    std::string(fn) + ": " + #call + ": " + cudaGetErrorString(e__) + " (the registry is unchanged)");                        \
                }                                                                                                                                              \
        } while (0)

static uint64_t perc_registry_bytes(const trn_ctx::PercBufs &B) {
        return B.d_queries.cap + B.d_ops.cap + B.d_pterms.cap + B.d_covers.cap + B.d_csr_off.cap + B.d_csr.cap + B.d_unanch.cap;
}

static void perc_refresh_info(trn_ctx::PercBufs &B) {
        B.info = trn_percolator_info{B.nlive, B.nunanchored, B.nnever, B.next_id, B.nentries, perc_registry_bytes(B)};
}

// The device half of an add (S: the added queries' plan, rebased onto the used program storage; their ids start at B.next_id) or a remove
// (removed: the bitmap of every removed id after the call; compact: rewrite the program storage without the removed queries).  nentries /
// nunanchored: the index's entries and the unanchored ids after the call (the host knows them from the per-id sizes).
static int perc_update(trn_ctx *c, const char *fn, const PercPlan *S, const std::vector<uint32_t> *removed, bool compact, uint64_t nentries,
                       uint32_t nunanchored) {
        auto &         B  = c->pq;
        const double   t0 = now_ms();
        const uint32_t nt = B.nterms, nq = B.next_id, nadd = S ? uint32_t(S->queries.size()) : 0u;
        // the added queries' anchor entries, by (term, id)
        std::vector<PercEntry> ne;
        std::vector<uint32_t>  nterm;
        if (S) {
                std::vector<std::pair<uint32_t, PercEntry>> e;
                e.reserve(S->covers.size());
                for (uint32_t q = 0; q < nadd; ++q)
                        for (uint32_t j = 0; j < S->queries[q].ncover; ++j)
                                e.push_back({S->covers[S->queries[q].cover_begin - B.cov_used + j], PercEntry{nq + q, j}});
                std::stable_sort(e.begin(), e.end(), [](const auto &a, const auto &b) { return a.first < b.first; });
                for (const auto &x : e) {
                        nterm.push_back(x.first);
                        ne.push_back(x.second);
                }
        }
        const uint64_t nold = B.nentries, nold_u = B.nunanchored, nnew = ne.size();
        const uint32_t nadd_u = S ? uint32_t(S->unanchored.size()) : 0u;
        if (!B.uev[0])
                for (Event &e : B.uev)
                        CKPU(cudaEventCreate(&e.h));
        cudaStream_t st = c->stream;
        auto         up = [&](DevBuf &b, const void *src, size_t n) -> cudaError_t {
                if (const cudaError_t e = b.ensure(std::max<size_t>(16, n)); e != cudaSuccess)
                        return e;
                return n ? cudaMemcpyAsync(b.p, src, n, cudaMemcpyHostToDevice, st) : cudaSuccess;
        };
        const uint64_t nmax = std::max<uint64_t>({nold, nold_u, nt, nq});
        CKPU(B.d_keep.ensure(std::max<size_t>(16, nmax * 4)));
        CKPU(B.d_kscan.ensure((nmax + 1) * 8));
        CKPU(B.d_upart.ensure((nmax / 4096 + 2) * 8));
        CKPU(B.d_cnt.ensure(std::max<size_t>(16, size_t(nt) * 4)));
        CKPU(B.d_toff.ensure((size_t(nt) + 1) * 8));
        DevBuf n_off, n_csr, n_un; // the rebuilt index and unanchored list
        CKPU(n_off.ensure((size_t(nt) + 1) * 4));
        CKPU(n_csr.ensure(std::max<size_t>(16, nentries * sizeof(PercEntry))));
        CKPU(n_un.ensure(std::max<size_t>(16, size_t(nunanchored) * 4)));
        const uint32_t *rm = nullptr;
        if (removed) {
                CKPU(up(B.d_removed, removed->data(), removed->size() * 4));
                rm = B.d_removed.as<uint32_t>();
        }
        CKPU(cudaEventRecord(B.uev[0], st));

        // ---- program storage: the added queries' programs behind the used ones (a full buffer is replaced by one twice its size), or the
        // live queries' programs compacted into buffers of their size
        DevBuf g_q, g_ops, g_pt, g_cov;
        uint64_t ops_used = B.ops_used, pt_used = B.pt_used, cov_used = B.cov_used;
        auto     append   = [&](DevBuf &cur, DevBuf &grown, size_t used, const void *src, size_t n) -> cudaError_t {
                DevBuf *dst = &cur;
                if (used + n > cur.cap) {
                        if (const cudaError_t e = grown.ensure(std::max(used + n, 2 * cur.cap)); e != cudaSuccess)
                                return e;
                        if (used)
                                if (const cudaError_t e = cudaMemcpyAsync(grown.p, cur.p, used, cudaMemcpyDeviceToDevice, st); e != cudaSuccess)
                                        return e;
                        dst = &grown;
                }
                return n ? cudaMemcpyAsync(static_cast<char *>(dst->p) + used, src, n, cudaMemcpyHostToDevice, st) : cudaSuccess;
        };
        if (S) {
                CKPU(append(B.d_queries, g_q, size_t(nq) * sizeof(PercQuery), S->queries.data(), S->queries.size() * sizeof(PercQuery)));
                CKPU(append(B.d_ops, g_ops, B.ops_used * sizeof(PercOp), S->ops.data(), S->ops.size() * sizeof(PercOp)));
                CKPU(append(B.d_pterms, g_pt, B.pt_used * 4, S->phrase_terms.data(), S->phrase_terms.size() * 4));
                CKPU(append(B.d_covers, g_cov, B.cov_used * 4, S->covers.data(), S->covers.size() * 4));
                ops_used += S->ops.size();
                pt_used += S->phrase_terms.size();
                cov_used += S->covers.size();
        } else if (compact) {
                ops_used = pt_used = cov_used = 0;
                for (uint32_t q = 0; q < nq; ++q)
                        if (!((*removed)[q >> 5] >> (q & 31u) & 1u)) {
                                ops_used += B.sizes[q].nops;
                                pt_used += B.sizes[q].npt;
                                cov_used += B.sizes[q].ncover;
                        }
                DevBuf c_n, c_s; // per id: its ops / phrase terms / cover terms, and their scans
                CKPU(c_n.ensure(std::max<size_t>(16, size_t(nq) * 12)));
                CKPU(c_s.ensure((size_t(nq) + 1) * 24));
                CKPU(g_q.ensure(std::max<size_t>(16, size_t(nq) * sizeof(PercQuery))));
                CKPU(g_ops.ensure(std::max<size_t>(16, ops_used * sizeof(PercOp))));
                CKPU(g_pt.ensure(std::max<size_t>(16, pt_used * 4)));
                CKPU(g_cov.ensure(std::max<size_t>(16, cov_used * 4)));
                uint32_t *          cn = c_n.as<uint32_t>();
                unsigned long long *cs = c_s.as<unsigned long long>();
                CKPU(launch_perc_upd_prog_sizes(B.d_queries.as<PercQuery>(), B.d_ops.as<PercOp>(), nq, rm, cn, cn + nq, cn + 2 * size_t(nq), st));
                for (int k = 0; k < 3; ++k)
                        CKPU(launch_enc_scan(cn + k * size_t(nq), nq, B.d_upart.as<unsigned long long>(), cs + k * (size_t(nq) + 1), st));
                CKPU(launch_perc_upd_prog_scatter(B.d_queries.as<PercQuery>(), B.d_ops.as<PercOp>(), B.d_pterms.as<uint32_t>(), B.d_covers.as<uint32_t>(), nq, rm,
                                                  cs, cs + (size_t(nq) + 1), cs + 2 * (size_t(nq) + 1), g_q.as<PercQuery>(), g_ops.as<PercOp>(),
                                                  g_pt.as<uint32_t>(), g_cov.as<uint32_t>(), st));
                CKPU(cudaStreamSynchronize(st)); // c_n / c_s are freed on return
        }

        // ---- the anchor index: surviving old entries of every term, then its new ones
        uint32_t *          keep  = B.d_keep.as<uint32_t>();
        unsigned long long *kscan = B.d_kscan.as<unsigned long long>(), *part = B.d_upart.as<unsigned long long>();
        CKPU(up(B.d_new, ne.data(), ne.size() * sizeof(PercEntry)));
        CKPU(up(B.d_new_terms, nterm.data(), nterm.size() * 4));
        CKPU(launch_perc_upd_keep(B.d_csr.as<PercEntry>(), nold, rm, keep, st));
        CKPU(launch_enc_scan(keep, nold, part, kscan, st));
        CKPU(launch_perc_upd_csr(B.d_csr.as<PercEntry>(), B.d_csr_off.as<uint32_t>(), nt, nold, keep, kscan, B.d_new.as<PercEntry>(),
                                 B.d_new_terms.as<uint32_t>(), uint32_t(nnew), B.d_cnt.as<uint32_t>(), part, B.d_toff.as<unsigned long long>(),
                                 n_csr.as<PercEntry>(), n_off.as<uint32_t>(), st));
        // ---- the unanchored list: its surviving ids, then the added ones
        CKPU(up(B.d_new_unanch, S ? S->unanchored.data() : nullptr, size_t(nadd_u) * 4));
        CKPU(launch_perc_upd_keep(B.d_unanch.as<uint32_t>(), nold_u, rm, keep, st));
        CKPU(launch_enc_scan(keep, nold_u, part, kscan, st));
        CKPU(launch_perc_upd_unanch(B.d_unanch.as<uint32_t>(), nold_u, keep, kscan, B.d_new_unanch.as<uint32_t>(), nadd_u, n_un.as<uint32_t>(), st));
        CKPU(cudaEventRecord(B.uev[1], st));
        CKPU(cudaStreamSynchronize(st));

        // ---- every step succeeded: the new buffers replace the old ones
        B.d_csr_off = std::move(n_off);
        B.d_csr     = std::move(n_csr);
        B.d_unanch  = std::move(n_un);
        const std::pair<DevBuf *, DevBuf *> grown[] = {{&g_q, &B.d_queries}, {&g_ops, &B.d_ops}, {&g_pt, &B.d_pterms}, {&g_cov, &B.d_covers}};
        for (const auto &[g, b] : grown)
                if (g->p)
                        *b = std::move(*g);
        B.nentries    = nentries;
        B.nunanchored = nunanchored;
        B.ops_used    = ops_used;
        B.pt_used     = pt_used;
        B.cov_used    = cov_used;
        (void)cudaEventElapsedTime(&B.update_ms, B.uev[0], B.uev[1]);
        B.update_host_ms = float(now_ms() - t0);
        return TRN_OK;
}

extern "C" int trn_percolator_add(trn_ctx *c, const trn_query *queries, uint32_t nq, uint32_t *first_id, trn_percolator_info *out) {
        static const char *fn = "trn_percolator_add";
        if (!c)
                return TRN_ERR_ARG;
        if (nq && !queries)
                return fail(c, TRN_ERR_ARG, "trn_percolator_add: bad arguments");
        auto &B = c->pq;
        if (!B.have)
                return fail(c, TRN_ERR_STATE, "trn_percolator_add: no query set registered (trn_percolator_register)");
        CK(cudaSetDevice(c->device));
        const uint32_t first = B.next_id;
        if (nq) {
                if (uint64_t(B.next_id) + nq > c->perc_max_ids)
                        return fail(c, TRN_ERR_CAPACITY, "trn_percolator_add: ids would reach " + std::to_string(c->perc_max_ids) + " (" +
                                                             std::to_string(B.next_id) + " issued; register the set again to start at 0)");
                PercPlan    S;
                std::string err;
                if (const int rc = perc_plan_queries(queries, nq, B.next_id, B.nterms, B.term_cost.empty() ? nullptr : B.term_cost.data(), S, err))
                        return fail(c, rc, "trn_percolator_add: " + err);
                if (B.nentries + S.covers.size() >= c->perc_max_entries || B.cov_used + S.covers.size() >= (1ull << 32) ||
                    B.ops_used + S.ops.size() >= (1ull << 32) || B.pt_used + S.phrase_terms.size() >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, "trn_percolator_add: the registry's anchor entries or program words would reach its limit (" +
                                                             std::to_string(B.nentries + S.covers.size()) + " anchor entries)");
                // rebase the slice onto the used program storage
                for (PercQuery &Q : S.queries) {
                        Q.op_begin += uint32_t(B.ops_used);
                        Q.cover_begin += uint32_t(B.cov_used);
                }
                for (PercOp &o : S.ops)
                        if (o.op == PERC_PHRASE)
                                o.term += uint32_t(B.pt_used);
                const uint64_t nentries = B.nentries + S.covers.size();
                const uint32_t nun      = B.nunanchored + uint32_t(S.unanchored.size());
                if (const int rc = perc_update(c, fn, &S, nullptr, false, nentries, nun))
                        return rc;
                for (uint32_t q = 0; q < nq; ++q)
                        B.sizes.push_back({S.queries[q].nops, S.npt[q], S.queries[q].ncover, S.status[q]});
                B.next_id += nq;
                B.removed.resize((size_t(B.next_id) + 31u) / 32u, 0u);
                B.nlive += nq;
                B.nnever += S.never;
        }
        if (first_id)
                *first_id = first;
        perc_refresh_info(B);
        if (out)
                *out = B.info;
        return TRN_OK;
}

extern "C" int trn_percolator_remove(trn_ctx *c, const uint32_t *ids, uint32_t n, trn_percolator_info *out) {
        static const char *fn = "trn_percolator_remove";
        if (!c)
                return TRN_ERR_ARG;
        if (n && !ids)
                return fail(c, TRN_ERR_ARG, "trn_percolator_remove: bad arguments");
        auto &B = c->pq;
        if (!B.have)
                return fail(c, TRN_ERR_STATE, "trn_percolator_remove: no query set registered (trn_percolator_register)");
        CK(cudaSetDevice(c->device));
        if (n) {
                std::vector<uint32_t> rem = B.removed;
                uint64_t              nentries = B.nentries, dead = B.dead_words;
                uint32_t              nun = B.nunanchored, nnever = B.nnever;
                for (uint32_t i = 0; i < n; ++i) {
                        const uint32_t q = ids[i];
                        if (q >= B.next_id)
                                return fail(c, TRN_ERR_ARG, "trn_percolator_remove: id " + std::to_string(q) + " was never issued (next id " + std::to_string(B.next_id) + ")");
                        if (rem[q >> 5] >> (q & 31u) & 1u)
                                return fail(c, TRN_ERR_ARG, "trn_percolator_remove: id " + std::to_string(q) +
                                                                (B.removed[q >> 5] >> (q & 31u) & 1u ? " was already removed" : " appears twice"));
                        rem[q >> 5] |= 1u << (q & 31u);
                        const auto &z = B.sizes[q];
                        if (z.status == PERC_ANCHORED)
                                nentries -= z.ncover;
                        nun -= z.status == PERC_UNANCHORED;
                        nnever -= z.status == PERC_NEVER;
                        dead += 2ull * z.nops + z.npt + z.ncover;
                }
                // compact when the removed queries' program words outnumber the live ones
                const uint64_t words   = 2ull * B.ops_used + B.pt_used + B.cov_used;
                const bool     compact = dead > words - dead;
                if (const int rc = perc_update(c, fn, nullptr, &rem, compact, nentries, nun))
                        return rc;
                B.removed    = std::move(rem);
                B.dead_words = compact ? 0 : dead;
                B.nlive -= n;
                B.nnever = nnever;
        }
        perc_refresh_info(B);
        if (out)
                *out = B.info;
        return TRN_OK;
}

extern "C" int trn_percolator_last_update(trn_ctx *c, float *device_ms, float *host_ms) {
        if (!c)
                return TRN_ERR_ARG;
        if (device_ms)
                *device_ms = c->pq.update_ms;
        if (host_ms)
                *host_ms = c->pq.update_host_ms;
        return TRN_OK;
}

extern "C" int trn_debug_percolator_registry(trn_ctx *c, uint32_t *csr_off, uint32_t *csr, uint64_t cap, uint32_t *unanchored, uint64_t ucap,
                                             uint32_t *nterms, uint64_t *nentries, uint64_t *nunanchored) {
        if (!c)
                return TRN_ERR_ARG;
        auto &B = c->pq;
        if (!B.have)
                return fail(c, TRN_ERR_STATE, "trn_debug_percolator_registry: no query set registered (trn_percolator_register)");
        if (nterms)
                *nterms = B.nterms;
        if (nentries)
                *nentries = B.nentries;
        if (nunanchored)
                *nunanchored = B.nunanchored;
        if ((csr && cap < B.nentries) || (unanchored && ucap < B.nunanchored))
                return fail(c, TRN_ERR_CAPACITY, "trn_debug_percolator_registry: " + std::to_string(B.nentries) + " entries and " +
                                                     std::to_string(B.nunanchored) + " unanchored ids do not fit");
        CK(cudaSetDevice(c->device));
        if (csr_off)
                CK(cudaMemcpyAsync(csr_off, B.d_csr_off.p, (size_t(B.nterms) + 1) * 4, cudaMemcpyDeviceToHost, c->stream));
        if (csr && B.nentries)
                CK(cudaMemcpyAsync(csr, B.d_csr.p, B.nentries * sizeof(PercEntry), cudaMemcpyDeviceToHost, c->stream));
        if (unanchored && B.nunanchored)
                CK(cudaMemcpyAsync(unanchored, B.d_unanch.p, size_t(B.nunanchored) * 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        return TRN_OK;
}

extern "C" int trn_debug_percolator_plan(const trn_query *queries, uint32_t nq, uint32_t nterms, const uint32_t *term_cost, uint8_t *status, uint32_t *cover_off,
                                         uint32_t *cover_terms, uint64_t cap, uint64_t *ncover, char *err, size_t errcap) {
        auto say = [&](const std::string &m) {
                if (err && errcap)
                        snprintf(err, errcap, "%s", m.c_str());
        };
        if ((nq && (!queries || !status)) || !cover_off || !ncover || (cap && !cover_terms)) {
                say("trn_debug_percolator_plan: bad arguments");
                return TRN_ERR_ARG;
        }
        PercPlan    P;
        std::string e;
        if (const int rc = perc_plan(queries, nq, nterms, term_cost, P, e)) {
                say(e);
                return rc;
        }
        *ncover = P.covers.size();
        if (P.covers.size() > cap) {
                say("trn_debug_percolator_plan: " + std::to_string(P.covers.size()) + " cover terms do not fit");
                return TRN_ERR_CAPACITY;
        }
        for (uint32_t q = 0; q < nq; ++q) {
                status[q]    = P.status[q];
                cover_off[q] = P.queries[q].cover_begin;
        }
        cover_off[nq] = uint32_t(P.covers.size());
        std::copy(P.covers.begin(), P.covers.end(), cover_terms);
        return TRN_OK;
}

// =================================================================================================== merge
// == MergeCandidatesCollection::commit() + merge() (merge.cpp): the plan on the host (mergeplan.h), the postings on the device (merge.cuh),
// the re-encoded terms through the device encoders in one call, the output assembled in output term order by one copy kernel.  One
// implementation behind both entry points: trn_merge_sources refuses a payload hit it has to re-encode, trn_merge_sources_payloads writes
// it (new_hit(pos, {payload, len}), merge.cpp:221-232, 352-361).
#define CKMG(call)                                                                                                                                             \
        do {                                                                                                                                                   \
                cudaError_t e__ = (call);                                                                                                                      \
                if (e__ == cudaErrorMemoryAllocation) {                                                                                                        \
                        cudaGetLastError();                                                                                                                    \
                        return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": working memory cannot be allocated on the device; merge fewer sources");    \
                }                                                                                                                                              \
                if (e__ != cudaSuccess) {                                                                                                                      \
                        c->err = std::string(#call) + ": " + cudaGetErrorString(e__);                                                                          \
                        return TRN_ERR_CUDA;                                                                                                                   \
                }                                                                                                                                              \
        } while (0)

static int merge_sources(trn_ctx *c, int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, trn_merged *out, bool payloads) {
        if (!c)
                return TRN_ERR_ARG;
        const char *const fn      = payloads ? "trn_merge_sources_payloads" : "trn_merge_sources";
        const double      t_begin = now_ms();
        if (!out)
                return fail(c, TRN_ERR_ARG, std::string(fn) + ": bad arguments");
        MergePlan   P;
        std::string perr;
        if (const int r = plan_merge(out_codec, src, n, disable_optimizations != 0, P, perr)) {
                const std::string planner_name = "trn_merge_sources"; // the name the planner's refusals start with
                if (payloads && perr.rfind(planner_name + ":", 0) == 0)
                        perr.replace(0, planner_name.size(), fn);
                return fail(c, r, perr);
        }
        const uint32_t nout = uint32_t(P.out.size() - 1);
        const auto     who  = [&](uint32_t s) { return std::string(fn) + ": source " + std::to_string(s) + " (generation " + std::to_string(src[s].generation) + ")"; };
        const auto     name = [&](uint32_t s, uint32_t t) { return who(s) + ", term [" + std::string(src[s].names[t]) + "]"; };
        CK(cudaSetDevice(c->device));
        auto &X = c->mg;
        for (auto &e : X.ev)
                if (!e)
                        CK(cudaEventCreate(&e.h));
        // ---- the sources' directories (host, as trn_upload_index / trn_upload_hits build them)
        std::vector<uint8_t>              used(n, 0);
        std::vector<BlockDirectory>       dirs(n);
        std::vector<HitsDirectory>        hdirs(n);
        std::vector<std::vector<DevTerm>> dts(n);
        for (const auto &p : P.parts)
                used[P.order[p.cand]] = 1;
        const int threads = int(std::max(1u, std::min(64u, std::thread::hardware_concurrency())));
        for (uint32_t s = 0; s < n; ++s) {
                if (!used[s])
                        continue;
                const auto &S = src[s];
                if (S.index_bytes >= (1ull << 32) || S.hits_bytes >= (1ull << 32))
                        return fail(c, TRN_ERR_ARG, who(s) + ": an index or hits.data of 4 GiB or more is not one source (range32_t offsets)");
                try {
                        build_directory(S.codec, S.index, S.index_bytes, S.terms, S.nterms, threads, dirs[s]);
                        dts[s] = dev_terms(dirs[s], S.terms, S.nterms);
                        if (S.codec == TRN_CODEC_LUCENE) {
                                std::vector<term_index_ctx> tc(S.nterms);
                                for (uint32_t i = 0; i < S.nterms; ++i)
                                        tc[i] = term_index_ctx{S.terms[i].documents, S.terms[i].chunk_off, S.terms[i].chunk_len};
                                build_hits_directory(S.index, S.index_bytes, S.hits, S.hits_bytes, tc.data(), S.nterms, dirs[s], threads, hdirs[s]);
                        }
                } catch (const std::bad_alloc &) {
                        return fail(c, TRN_ERR_CAPACITY, who(s) + ": out of host memory while building its directories");
                } catch (const std::exception &e) {
                        return fail(c, TRN_ERR_ARG, who(s) + ": " + e.what());
                }
                if (S.codec == TRN_CODEC_GOOGLE && dirs[s].block_docs && dirs[s].block_docs != Codecs::Google::N)
                        return fail(c, TRN_ERR_ARG, who(s) + ": GOOGLE blocks of " + std::to_string(dirs[s].block_docs) + " documents (the format's are 32)");
        }
        // ---- lists: every participant of every output term, term after term, newest first
        std::vector<MergeList>          lists;
        std::vector<unsigned long long> list_blk{0}, list_post{0}, re_first; // re_first: the first posting of each re-encoded term
        uint32_t                        maxdoc{0};
        for (uint32_t k = 0; k < nout; ++k) {
                const uint32_t b = P.out[k].part_begin, e = P.out[k + 1].part_begin;
                if (P.out[k].route == MERGE_REENCODE)
                        re_first.push_back(list_post.back());
                for (uint32_t q = b; q < e; ++q) {
                        const uint32_t s = P.order[P.parts[q].cand], t = P.parts[q].term;
                        MergeList      L{};
                        L.t        = dts[s][t];
                        L.view     = s;
                        L.term     = t;
                        L.cand     = P.parts[q].cand;
                        L.rank     = q - b;
                        L.nparts   = e - b;
                        L.reencode = P.out[k].route == MERGE_REENCODE;
                        lists.push_back(L);
                        list_blk.push_back(list_blk.back() + L.t.nblocks);
                        list_post.push_back(list_post.back() + L.t.documents);
                        maxdoc = std::max(maxdoc, L.t.last_doc);
                }
        }
        const uint32_t nlists = uint32_t(lists.size());
        const uint64_t nposts = list_post.back(), nblocks = list_blk.back();
        const uint32_t nre    = uint32_t(re_first.size());
        re_first.push_back(nposts);
        // ---- upload: every used source's bytes and directories, one view per source
        DevBuf   d_idx, d_hits, d_bl, d_bo, d_tf, d_hb, d_hbo, d_ht, d_views, d_lists, d_lblk, d_lpost, d_ud, d_uf, d_doc, d_fr, d_hc, d_hoff, d_pos, d_keep, d_ks,
            d_bm, d_part, d_odoc, d_ofr, d_osrc, d_ohoff, d_opos, d_err, d_cnt, d_idx2, d_tb, d_th, d_enc, d_henc, d_segs, d_oi, d_oh, d_pl, d_pv, d_opl, d_opv;
        std::vector<uint64_t> ibase(n + 1, 0), hbase(n + 1, 0), dbase(n + 1, 0), tbase(n + 1, 0), hbbase(n + 1, 0), termbase(n + 1, 0);
        for (uint32_t s = 0; s < n; ++s) {
                const bool u = used[s];
                ibase[s + 1]    = ibase[s] + (u ? (src[s].index_bytes + 511) / 256 * 256 : 0);
                hbase[s + 1]    = hbase[s] + (u && src[s].codec == TRN_CODEC_LUCENE ? (src[s].hits_bytes + 511) / 256 * 256 : 0);
                dbase[s + 1]    = dbase[s] + dirs[s].blk_last.size();
                tbase[s + 1]    = tbase[s] + dirs[s].tile_first.size();
                hbbase[s + 1]   = hbbase[s] + hdirs[s].hblk_off.size();
                termbase[s + 1] = termbase[s] + hdirs[s].hb_begin.size();
        }
        CKMG(d_idx.ensure(std::max<uint64_t>(256, ibase[n])));
        CKMG(d_hits.ensure(std::max<uint64_t>(256, hbase[n])));
        CKMG(d_bl.ensure(std::max<uint64_t>(4, dbase[n] * 4)));
        CKMG(d_bo.ensure(std::max<uint64_t>(4, dbase[n] * 4)));
        CKMG(d_hb.ensure(std::max<uint64_t>(4, dbase[n] * 4)));
        CKMG(d_tf.ensure(std::max<uint64_t>(4, tbase[n] * 4)));
        CKMG(d_hbo.ensure(std::max<uint64_t>(4, hbbase[n] * 4)));
        CKMG(d_ht.ensure(std::max<uint64_t>(8, termbase[n] * 8)));
        CK(cudaMemsetAsync(d_idx.p, 0, std::max<uint64_t>(256, ibase[n]), c->stream));
        CK(cudaMemsetAsync(d_hits.p, 0, std::max<uint64_t>(256, hbase[n]), c->stream));
        std::vector<HitsView>             views(std::max(1u, n));
        std::vector<std::vector<HitTerm>> hterms(n); // read by the asynchronous uploads until the stream synchronises
        for (uint32_t s = 0; s < n; ++s) {
                if (!used[s])
                        continue;
                const auto &S = src[s];
                const auto &D = dirs[s];
                const auto &H = hdirs[s];
                if (S.index_bytes)
                        CK(cudaMemcpyAsync(d_idx.as<uint8_t>() + ibase[s], S.index, S.index_bytes, cudaMemcpyHostToDevice, c->stream));
                if (S.codec == TRN_CODEC_LUCENE && S.hits_bytes)
                        CK(cudaMemcpyAsync(d_hits.as<uint8_t>() + hbase[s], S.hits, S.hits_bytes, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_bl.as<uint32_t>() + dbase[s], D.blk_last.data(), D.blk_last.size() * 4, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_bo.as<uint32_t>() + dbase[s], D.blk_off.data(), D.blk_off.size() * 4, cudaMemcpyHostToDevice, c->stream));
                if (!D.tile_first.empty())
                        CK(cudaMemcpyAsync(d_tf.as<uint32_t>() + tbase[s], D.tile_first.data(), D.tile_first.size() * 4, cudaMemcpyHostToDevice, c->stream));
                if (S.codec == TRN_CODEC_LUCENE) {
                        std::vector<HitTerm> &ht = hterms[s];
                        ht.resize(H.hb_begin.size());
                        for (size_t i = 0; i < ht.size(); ++i)
                                ht[i] = HitTerm{H.hb_begin[i], H.sum_hits[i]};
                        if (!H.hit_base.empty())
                                CK(cudaMemcpyAsync(d_hb.as<uint32_t>() + dbase[s], H.hit_base.data(), H.hit_base.size() * 4, cudaMemcpyHostToDevice, c->stream));
                        if (!H.hblk_off.empty())
                                CK(cudaMemcpyAsync(d_hbo.as<uint32_t>() + hbbase[s], H.hblk_off.data(), H.hblk_off.size() * 4, cudaMemcpyHostToDevice, c->stream));
                        if (!ht.empty())
                                CK(cudaMemcpyAsync(d_ht.as<HitTerm>() + termbase[s], ht.data(), ht.size() * 8, cudaMemcpyHostToDevice, c->stream));
                }
                views[s] = HitsView{d_idx.as<uint8_t>() + ibase[s], d_bl.as<uint32_t>() + dbase[s], d_bo.as<uint32_t>() + dbase[s], d_tf.as<uint32_t>() + tbase[s],
                                    d_hits.as<uint8_t>() + hbase[s], d_hb.as<uint32_t>() + dbase[s],  d_hbo.as<uint32_t>() + hbbase[s], d_ht.as<HitTerm>() + termbase[s],
                                    S.codec};
        }
        const uint64_t nupd   = P.upd_docid.size();
        const uint64_t nwords = (uint64_t(maxdoc) >> 5) + 1;
        CKMG(d_views.ensure(views.size() * sizeof(HitsView)));
        CKMG(d_lists.ensure(std::max<size_t>(1, nlists) * sizeof(MergeList)));
        CKMG(d_lblk.ensure((size_t(nlists) + 1) * 8));
        CKMG(d_lpost.ensure((size_t(nlists) + 1) * 8));
        CKMG(d_ud.ensure(std::max<uint64_t>(4, nupd * 4)));
        CKMG(d_uf.ensure(std::max<uint64_t>(4, nupd * 4)));
        CKMG(d_doc.ensure(std::max<uint64_t>(4, nposts * 4)));
        CKMG(d_fr.ensure(std::max<uint64_t>(4, nposts * 4)));
        CKMG(d_hc.ensure(std::max<uint64_t>(4, nposts * 4)));
        CKMG(d_hoff.ensure((nposts + 1) * 8));
        CKMG(d_keep.ensure(std::max<uint64_t>(4, nposts * 4)));
        CKMG(d_ks.ensure((nposts + 1) * 8));
        CKMG(d_part.ensure((nposts / 4096 + 4) * 8));
        CKMG(d_bm.ensure(nwords * 4));
        CKMG(d_err.ensure(24));
        CKMG(d_cnt.ensure(8));
        CKMG(d_idx2.ensure((size_t(nre) + 1) * 8));
        CKMG(d_tb.ensure((size_t(nre) + 1) * 8));
        CKMG(d_th.ensure((size_t(nre) + 1) * 8));
        CK(cudaMemcpyAsync(d_views.p, views.data(), views.size() * sizeof(HitsView), cudaMemcpyHostToDevice, c->stream));
        if (nlists)
                CK(cudaMemcpyAsync(d_lists.p, lists.data(), nlists * sizeof(MergeList), cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_lblk.p, list_blk.data(), (size_t(nlists) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_lpost.p, list_post.data(), (size_t(nlists) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        if (nupd) {
                CK(cudaMemcpyAsync(d_ud.p, P.upd_docid.data(), nupd * 4, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_uf.p, P.upd_first.data(), nupd * 4, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaMemcpyAsync(d_idx2.p, re_first.data(), (size_t(nre) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemsetAsync(d_bm.p, 0, nwords * 4, c->stream));
        CK(cudaMemsetAsync(d_err.p, 0xff, 24, c->stream));
        CK(cudaMemsetAsync(d_cnt.p, 0, 8, c->stream));
        MergeParams M{};
        M.views     = d_views.as<HitsView>();
        M.lists     = d_lists.as<MergeList>();
        M.nlists    = nlists;
        M.list_blk  = d_lblk.as<unsigned long long>();
        M.list_post = d_lpost.as<unsigned long long>();
        M.nblocks   = nblocks;
        M.nposts    = nposts;
        M.docids    = d_doc.as<uint32_t>();
        M.freqs     = d_fr.as<uint32_t>();
        M.hcount    = d_hc.as<uint32_t>();
        M.hoff      = d_hoff.as<unsigned long long>();
        M.upd_docid = d_ud.as<uint32_t>();
        M.upd_first = d_uf.as<uint32_t>();
        M.nupd      = nupd;
        M.keep      = d_keep.as<uint32_t>();
        M.bitmap    = d_bm.as<uint32_t>();
        M.kscan     = d_ks.as<unsigned long long>();
        M.error     = d_err.as<unsigned long long>();
        // ---- decode docIDs and freqs of every list; keep (which also drops the hits of every posting that is not written); the hits of
        // the kept postings, and again with their payloads when one of them carries one and the call takes them
        uint64_t nhits{0}, nkept{0}, herr[3]{~0ull, ~0ull, ~0ull}, docs_cnt{0};
        float    dec_ms{0}, m1{0}, m2{0}, d2{0}, enc_ms{0}, asm_ms{0};
        CK(cudaEventRecord(X.ev[0], c->stream));
        CK(launch_merge_decode(M, c->stream));
        CK(cudaEventRecord(X.ev[1], c->stream));
        CK(launch_merge_keep(M, c->stream));
        CK(launch_enc_scan(M.keep, nposts, d_part.as<unsigned long long>(), d_ks.as<unsigned long long>(), c->stream));
        CK(launch_merge_popcount(M.bitmap, nwords, d_cnt.as<unsigned long long>(), c->stream));
        CK(launch_merge_gather(M.kscan, d_idx2.as<unsigned long long>(), nre + 1, d_tb.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(X.ev[2], c->stream));
        CK(launch_enc_scan(M.hcount, nposts, d_part.as<unsigned long long>(), d_hoff.as<unsigned long long>(), c->stream));
        CK(cudaMemcpyAsync(&nhits, d_hoff.as<unsigned long long>() + nposts, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CKMG(d_pos.ensure(std::max<uint64_t>(4, nhits * 4)));
        M.positions = d_pos.as<uint32_t>();
        CK(launch_merge_hits_decode(M, false, c->stream));
        CK(cudaEventRecord(X.ev[3], c->stream));
        std::vector<uint64_t> h_tb(size_t(nre) + 1), h_th(size_t(nre) + 1);
        CK(cudaMemcpyAsync(h_tb.data(), d_tb.p, (size_t(nre) + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(herr, d_err.p, 24, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&docs_cnt, d_cnt.p, 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&dec_ms, X.ev[0], X.ev[1]));
        CK(cudaEventElapsedTime(&m1, X.ev[1], X.ev[2]));
        CK(cudaEventElapsedTime(&d2, X.ev[2], X.ev[3]));
        dec_ms += d2;
        const auto posting_name = [&](uint64_t i) {
                const MergeList &L = lists[uint32_t(std::upper_bound(list_post.begin(), list_post.end(), i) - list_post.begin()) - 1u];
                return name(L.view, L.term);
        };
        if (!payloads) {
                if (herr[0] != ~0ull)
                        return fail(c, TRN_ERR_UNSUPPORTED, posting_name(herr[0]) + ": a hit with a payload must be re-encoded; the device encoders write no payloads");
                if (herr[1] != ~0ull)
                        return fail(c, TRN_ERR_UNSUPPORTED,
                                    posting_name(herr[1]) + ": a hit at position 0 or above 16383 must be re-encoded; the device encoders take positions 1..16383");
        } else {
                if (herr[2] != ~0ull)
                        return fail(c, TRN_ERR_FORMAT, posting_name(herr[2]) + ": a hit stores a payload of more than 8 bytes (a payload is a u64)");
                if (herr[1] != ~0ull)
                        return fail(c, TRN_ERR_UNSUPPORTED, posting_name(herr[1]) + ": a hit at position 0 without a payload, or above 16383, must be re-encoded; "
                                                                                     "the device encoders take positions 1..16383 (0 with a payload)");
        }
        const bool with_payloads = payloads && herr[0] != ~0ull;
        if (with_payloads) {
                CKMG(d_pl.ensure(std::max<uint64_t>(4, nhits)));
                CKMG(d_pv.ensure(std::max<uint64_t>(8, nhits * 8)));
                M.plens = d_pl.as<uint8_t>();
                M.pays  = d_pv.as<unsigned long long>();
                CK(cudaEventRecord(X.ev[6], c->stream));
                CK(launch_merge_hits_decode(M, true, c->stream));
                CK(cudaEventRecord(X.ev[7], c->stream));
                CK(cudaStreamSynchronize(c->stream));
                CK(cudaEventElapsedTime(&d2, X.ev[6], X.ev[7]));
                dec_ms += d2;
        }
        nkept = h_tb[nre];
        CKMG(d_odoc.ensure(std::max<uint64_t>(4, nkept * 4)));
        CKMG(d_ofr.ensure(std::max<uint64_t>(4, nkept * 4)));
        CKMG(d_osrc.ensure(std::max<uint64_t>(8, nkept * 8)));
        CKMG(d_ohoff.ensure((nkept + 1) * 8));
        CKMG(d_part.ensure((std::max(nposts, nkept) / 4096 + 4) * 8));
        M.out_docids = d_odoc.as<uint32_t>();
        M.out_freqs  = d_ofr.as<uint32_t>();
        M.out_src    = d_osrc.as<unsigned long long>();
        M.out_hoff   = d_ohoff.as<unsigned long long>();
        CK(cudaEventRecord(X.ev[4], c->stream));
        CK(launch_merge_scatter(M, c->stream));
        CK(launch_enc_scan(M.out_freqs, nkept, d_part.as<unsigned long long>(), d_ohoff.as<unsigned long long>(), c->stream));
        CK(launch_merge_gather(M.out_hoff, d_tb.as<unsigned long long>(), nre + 1, d_th.as<unsigned long long>(), c->stream));
        CK(cudaMemcpyAsync(h_th.data(), d_th.p, (size_t(nre) + 1) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CKMG(d_opos.ensure(std::max<uint64_t>(4, h_th[nre] * 4)));
        M.out_positions = d_opos.as<uint32_t>();
        if (with_payloads) {
                CKMG(d_opl.ensure(std::max<uint64_t>(4, h_th[nre])));
                CKMG(d_opv.ensure(std::max<uint64_t>(8, h_th[nre] * 8)));
                M.out_plens = d_opl.as<uint8_t>();
                M.out_pays  = d_opv.as<unsigned long long>();
        }
        CK(launch_merge_out_hits(M, nkept, with_payloads, c->stream));
        CK(cudaEventRecord(X.ev[5], c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&m2, X.ev[4], X.ev[5]));
        for (DevBuf *b : {&d_fr, &d_hc, &d_hoff, &d_pos, &d_keep, &d_ks, &d_bm, &d_osrc, &d_lists, &d_lblk, &d_lpost, &d_ud, &d_uf, &d_pl, &d_pv})
                b->release();
        // ---- encode every re-encoded term in one call (orphans included: their headers are part of the output)
        std::vector<uint64_t> chunk, toff, hto;
        uint64_t              enc_bytes{0}, enc_hbytes{0};
        if (nre) {
                DevPostings DP{h_tb.data(), nre, d_tb.as<unsigned long long>(), M.out_docids, M.out_freqs, M.out_positions};
                if (with_payloads) {
                        DP.plens    = M.out_plens;
                        DP.payloads = M.out_pays;
                }
                int               r;
                if (out_codec == TRN_CODEC_GOOGLE) {
                        uint64_t nb{0};
                        r = encode_google_device(c, DP, Codecs::Google::N, Codecs::Google::SKIPLIST_STEP, P.countdown_phase, true, ~0ull, &enc_bytes, d_enc, chunk, toff,
                                                 &nb, &enc_ms);
                } else
                        r = encode_lucene_device(c, DP, true, ~0ull, &enc_bytes, true, ~0ull, &enc_hbytes, d_enc, d_henc, toff, &enc_ms, &hto);
                if (r == TRN_ERR_CUDA && c->err.find("out of memory") != std::string::npos)
                        return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": working memory cannot be allocated on the device; merge fewer sources");
                if (r == TRN_ERR_ARG || r == TRN_ERR_CAPACITY) { // the encoder's refusal, for the re-encoded terms as a whole: name the first
                        uint32_t k = 0;
                        while (P.out[k].route != MERGE_REENCODE)
                                ++k;
                        const MergePart &p0 = P.parts[P.out[k].part_begin];
                        return fail(c, r, std::string(fn) + ": re-encoding the merged terms (the first [" + std::string(src[P.order[p0.cand]].names[p0.term]) +
                                                  "] of " + who(P.order[p0.cand]) + "): " + c->err);
                }
                if (r)
                        return r;
        }
        // ---- assembly: output term order, appended chunks from the sources' bytes, re-encoded ones from the encoder's output
        const bool             lucene = out_codec == TRN_CODEC_LUCENE;
        std::vector<MergeCopy> segs;
        std::vector<trn_term>  terms;
        std::vector<uint32_t>  tsrc, tidx;
        uint64_t               io{0}, ho{0}, sum_docs{0}, sum_hits{0};
        uint32_t               appended{0}, reencoded{0}, orphaned{0};
        for (uint32_t k = 0, r = 0; k < nout; ++k) {
                const MergePart &p0 = P.parts[P.out[k].part_begin];
                const uint32_t   s0 = P.order[p0.cand];
                uint64_t         len, hlen, docs;
                const uint8_t   *isrc, *hsrc;
                if (P.out[k].route == MERGE_APPEND) {
                        const trn_term &T = src[s0].terms[p0.term];
                        len               = T.chunk_len;
                        docs              = T.documents;
                        isrc              = d_idx.as<uint8_t>() + ibase[s0] + T.chunk_off;
                        hlen              = 0;
                        hsrc              = nullptr;
                        if (lucene) {
                                if (len < 14)
                                        return fail(c, TRN_ERR_ARG, name(s0, p0.term) + ": a LUCENE chunk is at least 14 bytes");
                                uint32_t hdo, pcs;
                                std::memcpy(&hdo, src[s0].index + T.chunk_off, 4);
                                std::memcpy(&pcs, src[s0].index + T.chunk_off + 8, 4);
                                if (uint64_t(hdo) + pcs > src[s0].hits_bytes)
                                        return fail(c, TRN_ERR_ARG, name(s0, p0.term) + ": its positions chunk lies outside the source's hits.data");
                                hlen = pcs;
                                hsrc = d_hits.as<uint8_t>() + hbase[s0] + hdo;
                        }
                        ++appended;
                } else {
                        len  = toff[r + 1] - toff[r];
                        isrc = d_enc.as<uint8_t>() + toff[r];
                        hlen = lucene ? hto[r + 1] - hto[r] : 0;
                        hsrc = lucene ? d_henc.as<uint8_t>() + hto[r] : nullptr;
                        docs = h_tb[r + 1] - h_tb[r];
                        if (P.out[k].stats) {
                                sum_docs += docs;
                                sum_hits += h_th[r + 1] - h_th[r];
                        }
                        ++r;
                        if (docs)
                                ++reencoded;
                        else
                                ++orphaned;
                }
                if (ho >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": the merged hits.data reaches 4 GiB (u32 hitsDataOffset)");
                // a CTA per piece of at most kPiece bytes, so a long chunk is copied by many CTAs
                constexpr uint64_t kPiece = 1u << 16;
                for (uint64_t a = 0; a < len || a == 0; a += kPiece)
                        segs.push_back(MergeCopy{isrc + a, io + a, std::min(kPiece, len - a), 0u, lucene && a == 0 ? 1u : 0u, uint32_t(ho)});
                for (uint64_t a = 0; a < hlen; a += kPiece)
                        segs.push_back(MergeCopy{hsrc + a, ho + a, std::min(kPiece, hlen - a), 1u, 0u, 0u});
                if (docs) {
                        terms.push_back(trn_term{uint32_t(docs), uint32_t(io), uint32_t(len)});
                        tsrc.push_back(s0);
                        tidx.push_back(p0.term);
                }
                io += len;
                ho += hlen;
                if (io >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": the merged index reaches 4 GiB (range32_t chunk offsets)");
        }
        if (ho >= (1ull << 32))
                return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": the merged hits.data reaches 4 GiB (u32 hitsDataOffset)");
        std::vector<uint8_t> index, hits;
        try {
                index.resize(io);
                hits.resize(ho);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, std::string(fn) + ": the result cannot be allocated on the host");
        }
        CKMG(d_segs.ensure(std::max<size_t>(1, segs.size()) * sizeof(MergeCopy)));
        CKMG(d_oi.ensure(std::max<uint64_t>(4, io)));
        CKMG(d_oh.ensure(std::max<uint64_t>(4, ho)));
        if (!segs.empty())
                CK(cudaMemcpyAsync(d_segs.p, segs.data(), segs.size() * sizeof(MergeCopy), cudaMemcpyHostToDevice, c->stream));
        CK(cudaEventRecord(X.ev[6], c->stream));
        CK(launch_merge_assemble(d_segs.as<MergeCopy>(), uint32_t(segs.size()), d_oi.as<uint8_t>(), d_oh.as<uint8_t>(), c->stream));
        CK(cudaEventRecord(X.ev[7], c->stream));
        if (io)
                CK(cudaMemcpyAsync(index.data(), d_oi.p, io, cudaMemcpyDeviceToHost, c->stream));
        if (ho)
                CK(cudaMemcpyAsync(hits.data(), d_oh.p, ho, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        CK(cudaEventElapsedTime(&asm_ms, X.ev[6], X.ev[7]));
        X.index.swap(index);
        X.hits.swap(hits);
        X.terms.swap(terms);
        X.term_source.swap(tsrc);
        X.term_index.swap(tidx);
        *out                  = trn_merged{};
        out->index            = X.index.data();
        out->index_bytes      = X.index.size();
        out->hits             = X.hits.data();
        out->hits_bytes       = X.hits.size();
        out->terms            = X.terms.data();
        out->term_source      = X.term_source.data();
        out->term_index       = X.term_index.data();
        out->nterms           = uint32_t(X.terms.size());
        out->total_terms      = uint32_t(X.terms.size());
        out->docs_cnt         = uint32_t(docs_cnt);
        out->sum_terms_docs   = sum_docs;
        out->sum_term_hits    = sum_hits;
        out->appended         = appended;
        out->reencoded        = reencoded;
        out->orphaned         = orphaned;
        out->postings_read    = nposts;
        out->postings_written = nkept;
        out->decode_ms        = dec_ms;
        out->merge_ms         = m1 + m2;
        out->encode_ms        = enc_ms;
        out->assemble_ms      = asm_ms;
        out->total_ms         = float(now_ms() - t_begin);
        c->have_kernel_events = false;
        return TRN_OK;
}

extern "C" int trn_merge_sources_payloads(trn_ctx *c, int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, trn_merged *out) {
        return merge_sources(c, out_codec, src, n, disable_optimizations, out, true);
}

extern "C" int trn_merge_sources(trn_ctx *c, int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, trn_merged *out) {
        return merge_sources(c, out_codec, src, n, disable_optimizations, out, false);
}

extern "C" int trn_debug_merge_plan(int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, uint32_t *order, uint8_t *route,
                                    uint8_t *stats, uint32_t *part_off, uint32_t *part_cand, uint32_t *part_term, uint32_t *nout, uint64_t *nparts,
                                    uint32_t *upd_docid, uint32_t *upd_first, uint64_t *nupd, uint32_t *countdown_phase, char *err, size_t errcap) {
        MergePlan   P;
        std::string e;
        const int   r = plan_merge(out_codec, src, n, disable_optimizations != 0, P, e);
        if (r) {
                if (err && errcap)
                        std::snprintf(err, errcap, "%s", e.c_str());
                return r;
        }
        const uint32_t no = uint32_t(P.out.size() - 1);
        for (uint32_t j = 0; j < n; ++j)
                order[j] = P.order[j];
        for (uint32_t k = 0; k <= no; ++k) {
                part_off[k] = P.out[k].part_begin;
                if (k < no) {
                        route[k] = P.out[k].route;
                        stats[k] = P.out[k].stats;
                }
        }
        for (size_t q = 0; q < P.parts.size(); ++q) {
                part_cand[q] = P.parts[q].cand;
                part_term[q] = P.parts[q].term;
        }
        for (size_t i = 0; i < P.upd_docid.size(); ++i) {
                upd_docid[i] = P.upd_docid[i];
                upd_first[i] = P.upd_first[i];
        }
        *nout            = no;
        *nparts          = P.parts.size();
        *nupd            = P.upd_docid.size();
        *countdown_phase = P.countdown_phase;
        return TRN_OK;
}
