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
#include "kernels.h"
#include "planner.h"
#include <algorithm>
#include <array>
#include <chrono>
#include <cmath>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <stdexcept>
#include <functional>
#include <map>
#include <string>
#include <unordered_map>
#include <thread>
#include <vector>

using namespace trn;

namespace {
struct DevBuf {
        void * p{nullptr};
        size_t cap{0};
        cudaError_t ensure(size_t bytes) {
                if (bytes <= cap)
                        return cudaSuccess;
                if (p)
                        cudaFree(p);
                p   = nullptr;
                cap = 0;
                size_t want = bytes + bytes / 8 + 256;
                cudaError_t e = cudaMalloc(&p, want);
                if (e == cudaSuccess)
                        cap = want;
                return e;
        }
        void release() {
                if (p)
                        cudaFree(p);
                p   = nullptr;
                cap = 0;
        }
        template <class T> T *as() const {
                return static_cast<T *>(p);
        }
};
struct PinBuf {
        void * p{nullptr};
        size_t cap{0};
        cudaError_t ensure(size_t bytes) {
                if (bytes <= cap)
                        return cudaSuccess;
                if (p)
                        cudaFreeHost(p);
                p   = nullptr;
                cap = 0;
                size_t want = bytes + bytes / 8 + 256;
                cudaError_t e = cudaHostAlloc(&p, want, cudaHostAllocDefault);
                if (e == cudaSuccess)
                        cap = want;
                return e;
        }
        void release() {
                if (p)
                        cudaFreeHost(p);
                p   = nullptr;
                cap = 0;
        }
        template <class T> T *as() const {
                return static_cast<T *>(p);
        }
};
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
        int                  flat_threads{320}; // TRN_SF_THREADS: CTA size of k_score_flat (256/320/384: two CTAs per SM; 512/640: one)
        uint64_t             index_bytes{0}, dir_bytes{0}, total_blocks{0}, total_postings{0};
        DevBuf               d_index, d_blk_last, d_blk_off, d_terms, d_tile_first, d_masked;
        bool                 have_masked{false};
        std::vector<DevTerm> h_terms;
        // batch scratch (grow-only)
        DevBuf d_queries, d_steps, d_small[2], d_item_off, d_item_cnt, d_item_dst, d_seg_docids, d_seg_scores, d_out_docids[2], d_out_scores[2], d_q_offsets[2], d_cand,
            d_topk_docids, d_topk_scores, d_topk_counts, d_fq, d_leaves, d_luts, d_dec_units, d_dec_a, d_dec_b, d_dec_c, d_dec_docids, d_dec_freqs, d_dec_sums, d_merge_docids, d_merge_scores;
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
        cudaEvent_t ev0{nullptr}, ev1{nullptr}, evk0{nullptr}, evk1{nullptr};
        bool        have_kernel_events{false};
        // pipelined host-buffer path (trn_exec_batch): kernels of chunk i+1 overlap the D2H of chunk i
        cudaStream_t copy_stream{nullptr};
        cudaEvent_t  ev_done[2]{nullptr, nullptr}, ev_d2h[2]{nullptr, nullptr}, ev_ck0[16]{}, ev_ck1[16]{};
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
        float    last_ms{0};
        std::vector<uint8_t> last_routes; // TRN_ROUTE_* of every query of the last batch (trn_debug_last_routes)
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
        CK(cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking));
        for (int i = 0; i < 2; ++i) {
                CK(cudaEventCreateWithFlags(&c->ev_done[i], cudaEventDisableTiming));
                CK(cudaEventCreateWithFlags(&c->ev_d2h[i], cudaEventDisableTiming));
        }
        for (int i = 0; i < 16; ++i) {
                CK(cudaEventCreate(&c->ev_ck0[i]));
                CK(cudaEventCreate(&c->ev_ck1[i]));
        }
        CK(cudaEventCreate(&c->ev0));
        CK(cudaEventCreate(&c->ev1));
        CK(cudaEventCreate(&c->evk0));
        CK(cudaEventCreate(&c->evk1));
        return TRN_OK;
}

extern "C" void trn_destroy(trn_ctx *c) {
        if (!c)
                return;
        cudaSetDevice(c->device);
        for (DevBuf *b : {&c->d_index, &c->d_blk_last, &c->d_blk_off, &c->d_terms, &c->d_tile_first, &c->d_masked, &c->d_queries, &c->d_steps, &c->d_small[0], &c->d_small[1], &c->d_item_off,
                          &c->d_item_cnt, &c->d_item_dst, &c->d_seg_docids, &c->d_seg_scores, &c->d_out_docids[0], &c->d_out_docids[1], &c->d_out_scores[0], &c->d_out_scores[1], &c->d_q_offsets[0], &c->d_q_offsets[1], &c->d_cand,
                          &c->d_topk_docids, &c->d_topk_scores, &c->d_topk_counts, &c->d_fq, &c->d_leaves, &c->d_luts, &c->d_dec_units, &c->d_dec_a, &c->d_dec_b, &c->d_dec_c, &c->d_dec_docids, &c->d_dec_freqs,
                          &c->d_dec_sums, &c->d_merge_docids, &c->d_merge_scores})
                b->release();
        for (PinBuf *b : {&c->h_offsets, &c->h_docids, &c->h_scores, &c->h_counts, &c->h_small, &c->h_chunk, &c->h_item_desc})
                b->release();
        for (cudaEvent_t e : {c->ev0, c->ev1, c->evk0, c->evk1, c->ev_done[0], c->ev_done[1], c->ev_d2h[0], c->ev_d2h[1]})
                if (e)
                        cudaEventDestroy(e);
        for (int i = 0; i < 16; ++i) {
                if (c->ev_ck0[i])
                        cudaEventDestroy(c->ev_ck0[i]);
                if (c->ev_ck1[i])
                        cudaEventDestroy(c->ev_ck1[i]);
        }
        if (c->copy_stream)
                cudaStreamDestroy(c->copy_stream);
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
        try {
                ht = dev_terms(dir, terms, nterms);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_index: out of host memory");
        }
        uint32_t min_docid;
        docid_span(ht, min_docid, max_docid);
        c->have_index   = false; // until the new index is completely in place
        c->pc.codec     = codec;
        c->pc.min_docid = min_docid;
        c->pc.max_docid = max_docid;
        c->block_docs   = dir.block_docs;
        c->nterms       = nterms;
        const uint32_t W = 1u << c->pc.tile_shift;
        c->ntiles       = uint32_t((uint64_t(max_docid) + 1 + W - 1) >> c->pc.tile_shift);
        c->h_terms      = std::move(ht);
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
        return ix;
}

// =================================================================================================== exec
// small device scratch layout (d_small): [0] ticket u32, [2..3] seg_cursor u64, [4] overflow u32, then per-query arrays.
// routes[0 .. nq): the TRN_ROUTE_* of every query (written on success)
static int exec_device_impl(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out, int set, cudaEvent_t k0, cudaEvent_t k1,
                            uint8_t *routes) {
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
        c->pc.allow_phrase     = c->pc.codec == TRN_CODEC_GOOGLE || c->have_hits; // GOOGLE: inline hits; LUCENE: hits.data uploaded (trn_upload_hits)
        BatchPlan   plan;
        std::string perr;
        const int   prc = plan_batch(c->pc, c->h_terms, queries, nq, mode, k, plan, perr);
        if (prc != TRN_OK)
                return fail(c, prc, perr);
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
        if (!steps.empty())
                CK(cudaMemcpyAsync(c->d_steps.p, steps.data(), steps.size() * sizeof(DevStep), cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemsetAsync(small, 0, smallBytes, c->stream));

        ExecParams P;
        std::memset(&P, 0, sizeof(P));
        P.ix           = dev_index(c);
        P.queries      = c->d_queries.as<DevQuery>();
        P.steps        = c->d_steps.as<DevStep>();
        P.nq           = nq;
        P.total_items  = totalItems;
        P.gen_items    = uint32_t(plan.gen_items);
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

        uint32_t launches{0};
        if (totalItems) {
                const bool     warpKernel = !scored;
                const uint64_t ownItems   = plan.gen_items; // tickets of the step-program launch
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
                        CK(launch_build_luts(S.leaves, uint32_t(plan.leaves.size()), c->d_luts.as<float>(), c->stream));
                        CK(launch_score_flat(S, c->flat_threads, c->num_sms, c->stream));
                        launches += 2;
                }
                if (ownItems) {
                        const int perSM = warpKernel ? exec_docs_max_ctas_per_sm(execShift, plan.nslots, exec_docs_stage_bytes(), false, c->pc.codec == TRN_CODEC_LUCENE) : exec_max_ctas_per_sm(execShift, plan.nslots, mode, c->pc.codec);
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
                        P2.ticket     = reinterpret_cast<uint32_t *>(small + 4);
                        const int perSM = exec_docs_max_ctas_per_sm(P2.exec_shift, P2.nslots, exec_docs_stage_bytes(), true);
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
        if (!c)
                return TRN_ERR_ARG;
        CK(cudaSetDevice(c->device));
        c->have_kernel_events = false;
        c->tm                 = trn_timings{};
        c->last_routes.clear();
        const double t0       = now_ms();
        CK(cudaEventRecord(c->ev0, c->stream));
        std::vector<uint8_t> routes(nq);
        const int            r = exec_device_impl(c, queries, nq, mode, k, out, 0, c->evk0, c->evk1, routes.data());
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
        c->last_ms = ms;
        return TRN_OK;
}

// Host-buffer entry point.  DOCS_ONLY / SCORED_ALL batches are split into chunks: the fused kernels of chunk i+1 run while the
// results of chunk i travel to the (pinned) host buffer on a second stream — the e2e time tends to max(kernels, D2H) instead of
// their sum.  Output-side device buffers are double-buffered (set = chunk parity); everything else is reused in stream order.
extern "C" int trn_exec_batch(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out) {
        if (!c || !out)
                return TRN_ERR_ARG;
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
                const int    r  = trn_exec_batch_device(c, queries, nq, mode, k, nullptr);
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
        auto grow = [&](PinBuf &b, size_t need, size_t keep) -> cudaError_t {
                if (need <= b.cap)
                        return cudaSuccess;
                void *      np{nullptr};
                const size_t want = need + need / 4 + 4096;
                cudaError_t e = cudaHostAlloc(&np, want, cudaHostAllocDefault);
                if (e != cudaSuccess)
                        return e;
                if (b.p && keep) {
                        // earlier chunks' D2H into the old block must have landed before it is copied
                        cudaStreamSynchronize(c->copy_stream);
                        std::memcpy(np, b.p, keep);
                }
                if (b.p)
                        cudaFreeHost(b.p);
                b.p   = np;
                b.cap = want;
                return cudaSuccess;
        };
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
                CK(grow(c->h_docids, need, running * 4));
                if (scored)
                        CK(grow(c->h_scores, need, running * 4));
                if (total) {
                        CK(cudaMemcpyAsync(c->h_docids.as<uint32_t>() + running, c->d_out_docids[set].p, total * 4, cudaMemcpyDeviceToHost, c->copy_stream));
                        if (scored)
                                CK(cudaMemcpyAsync(c->h_scores.as<float>() + running, c->d_out_scores[set].p, total * 4, cudaMemcpyDeviceToHost, c->copy_stream));
                }
                if (compact) { // the chunk's segment descriptors; its queries' item ranges move behind the earlier chunks' items
                        const uint32_t ni = chunkItems[j];
                        CK(grow(c->h_item_desc, std::max<size_t>(4, std::max<uint64_t>(runningItems + ni, c->last_items_hint) * 4), runningItems * 4));
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
                const int  r = exec_device_impl(c, queries + ch[i].q0, ch[i].n, mode, k, &part, set, c->ev_ck0[i % 16], c->ev_ck1[i % 16], routes.data() + ch[i].q0);
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

extern "C" int trn_debug_plan(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid,
                              const trn_query *queries, uint32_t nq, int mode, uint32_t k, uint8_t *routes, uint32_t *nslots, char *err, size_t errcap) {
        auto seterr = [&](const std::string &m, int rc) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return rc;
        };
        if (!index || !terms || !queries || !nq || !routes || !nslots || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || mode < 0 || mode > 3)
                return seterr("bad arguments", TRN_ERR_ARG);
        BlockDirectory       dir;
        std::vector<DevTerm> ht;
        try {
                build_directory(codec, index, nbytes, terms, nterms, 1, dir);
                ht = dev_terms(dir, terms, nterms);
        } catch (const std::exception &e) {
                return seterr(e.what(), TRN_ERR_FORMAT);
        }
        PlanConfig pc   = initial_plan_config();
        pc.codec        = codec;
        pc.allow_phrase = codec == TRN_CODEC_GOOGLE;
        docid_span(ht, pc.min_docid, max_docid);
        pc.max_docid = max_docid;
        BatchPlan   plan;
        std::string perr;
        const int   rc = plan_batch(pc, ht, queries, nq, mode, k, plan, perr);
        if (rc != TRN_OK)
                return seterr(perr, rc);
        for (uint32_t q = 0; q < nq; ++q)
                routes[q] = uint8_t(plan.queries[q].route);
        nslots[0] = plan.nslots;
        nslots[1] = plan.tree_slots;
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
extern "C" int trn_encode_google(trn_ctx *c, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                                 uint32_t block_docs, uint32_t skiplist_step, uint32_t *countdown, uint8_t *out, uint64_t cap, uint64_t *out_bytes, trn_term *terms,
                                 float *device_ms) {
        if (!c)
                return TRN_ERR_ARG;
        if (!term_begin || !nterms || !out_bytes || !terms || block_docs == 0 || block_docs > 128 || skiplist_step == 0 ||
            (countdown && (*countdown == 0 || *countdown > skiplist_step)))
                return fail(c, TRN_ERR_ARG, "trn_encode_google: bad arguments");
        const uint64_t nposts = term_begin[nterms];
        if (term_begin[0] != 0 || (nposts && (!docids || !freqs)))
                return fail(c, TRN_ERR_ARG, "trn_encode_google: bad arguments");
        CK(cudaSetDevice(c->device));
        std::vector<uint64_t> blk_begin(nterms + 1);
        uint64_t              nblocks{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                if (term_begin[t + 1] < term_begin[t] || term_begin[t + 1] - term_begin[t] > 0xffffffffull)
                        return fail(c, TRN_ERR_ARG, "trn_encode_google: term_begin must ascend (at most 2^32 - 1 documents per term)");
                blk_begin[t] = nblocks;
                nblocks += (term_begin[t + 1] - term_begin[t] + block_docs - 1) / block_docs;
        }
        blk_begin[nterms] = nblocks;
        uint64_t nhits{0};
        if (positions)
                for (uint64_t i = 0; i < nposts; ++i)
                        nhits += freqs[i];
        const uint32_t phase0 = countdown ? (skiplist_step - *countdown) % skiplist_step : 0u;
        DevBuf d_tb, d_bb, d_doc, d_fr, d_pos, d_hb, d_bsz, d_bterm, d_boff, d_part, d_toff, d_cb, d_out, d_err;
        struct Free {
                std::vector<DevBuf *> v;
                ~Free() {
                        for (auto b : v)
                                b->release();
                }
        } fr{{&d_tb, &d_bb, &d_doc, &d_fr, &d_pos, &d_hb, &d_bsz, &d_bterm, &d_boff, &d_part, &d_toff, &d_cb, &d_out, &d_err}};
        const size_t parts = size_t(std::max(nposts, nblocks) / 4096 + 4);
        CK(d_tb.ensure((size_t(nterms) + 1) * 8));
        CK(d_bb.ensure((size_t(nterms) + 1) * 8));
        CK(d_doc.ensure(std::max<size_t>(4, nposts * 4)));
        CK(d_fr.ensure(std::max<size_t>(4, nposts * 4)));
        CK(d_bsz.ensure(std::max<size_t>(4, nblocks * 4)));
        CK(d_bterm.ensure(std::max<size_t>(4, nblocks * 4)));
        CK(d_boff.ensure((nblocks + 1) * 8));
        CK(d_part.ensure(parts * 8));
        CK(d_toff.ensure((size_t(nterms) + 1) * 8));
        CK(d_cb.ensure(size_t(nterms) * 8));
        CK(d_err.ensure(4));
        CK(cudaMemcpyAsync(d_tb.p, term_begin, (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(d_bb.p, blk_begin.data(), (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        if (nposts) {
                CK(cudaMemcpyAsync(d_doc.p, docids, nposts * 4, cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(d_fr.p, freqs, nposts * 4, cudaMemcpyHostToDevice, c->stream));
        }
        if (positions) {
                CK(d_pos.ensure(std::max<size_t>(4, nhits * 4)));
                CK(d_hb.ensure((nposts + 1) * 8));
                if (nhits)
                        CK(cudaMemcpyAsync(d_pos.p, positions, nhits * 4, cudaMemcpyHostToDevice, c->stream));
        }
        CK(cudaMemsetAsync(d_err.p, 0, 4, c->stream));
        EncParams E{};
        E.term_begin    = d_tb.as<unsigned long long>();
        E.blk_begin     = d_bb.as<unsigned long long>();
        E.nterms        = nterms;
        E.nblocks       = nblocks;
        E.docids        = d_doc.as<uint32_t>();
        E.freqs         = d_fr.as<uint32_t>();
        E.positions     = positions ? d_pos.as<uint32_t>() : nullptr;
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
                CK(launch_enc_scan(d_fr.as<uint32_t>(), nposts, d_part.as<unsigned long long>(), d_hb.as<unsigned long long>(), c->stream));
        CK(launch_enc_google_sizes(E, c->stream));
        CK(launch_enc_scan(d_bsz.as<uint32_t>(), nblocks, d_part.as<unsigned long long>(), d_boff.as<unsigned long long>(), c->stream));
        CK(launch_enc_term_sizes(E, d_cb.as<unsigned long long>(), c->stream));
        CK(cudaEventRecord(e1, c->stream));
        // chunk offsets: a prefix sum over the terms on the host (the output size must be known here anyway)
        std::vector<uint64_t> chunk(nterms), toff(nterms + 1);
        uint32_t              herr{0};
        CK(cudaMemcpyAsync(chunk.data(), d_cb.p, size_t(nterms) * 8, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaMemcpyAsync(&herr, d_err.p, 4, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        if (herr)
                return fail(c, TRN_ERR_ARG, "google encoder: document IDs must be > 0 and strictly ascending, positions in 1..16383 and non-decreasing");
        uint64_t total{0};
        for (uint32_t t = 0; t < nterms; ++t) {
                toff[t] = total;
                total += chunk[t];
        }
        toff[nterms] = total;
        *out_bytes   = total;
        if (total >= (1ull << 32))
                return fail(c, TRN_ERR_CAPACITY, "google encoder: the index of one source is limited to 4 GiB (range32_t, codecs.h:17-55)");
        if (total > cap || !out)
                return fail(c, TRN_ERR_CAPACITY, "trn_encode_google: output buffer too small");
        CK(d_out.ensure(std::max<size_t>(4, total)));
        E.out = d_out.as<uint8_t>();
        CK(cudaMemcpyAsync(d_toff.p, toff.data(), (size_t(nterms) + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaEventRecord(e2, c->stream));
        CK(cudaMemsetAsync(d_out.p, 0, std::max<size_t>(4, total), c->stream)); // a term without documents is its zero u16
        CK(launch_enc_google_write(E, c->stream));
        CK(cudaEventRecord(e3, c->stream));
        CK(cudaMemcpyAsync(out, d_out.p, total, cudaMemcpyDeviceToHost, c->stream));
        CK(cudaStreamSynchronize(c->stream));
        for (uint32_t t = 0; t < nterms; ++t) {
                terms[t].documents = uint32_t(term_begin[t + 1] - term_begin[t]);
                terms[t].chunk_off = uint32_t(toff[t]);
                terms[t].chunk_len = uint32_t(chunk[t]);
        }
        if (countdown)
                *countdown = skiplist_step - uint32_t((uint64_t(phase0) + nblocks) % skiplist_step);
        if (device_ms) {
                float a{0}, b{0};
                CK(cudaEventElapsedTime(&a, e0, e1));
                CK(cudaEventElapsedTime(&b, e2, e3));
                *device_ms = a + b;
        }
        c->have_kernel_events = false;
        return TRN_OK;
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
        // TRN_DECODE_KERNEL=legacy | single-pass: the round-1 kernels (register-staged span copy / cp.async lane gather), kept for A/B runs;
        // default: the bulk-copy streaming kernels of decode_stream.cuh
        static const std::string decodeKernel = getenv("TRN_DECODE_KERNEL") ? getenv("TRN_DECODE_KERNEL") : "";
        const bool               legacyDecode = (decodeKernel == "legacy" || decodeKernel == "single-pass") && c->block_docs == (c->pc.codec == TRN_CODEC_GOOGLE ? 32u : 128u);
        std::vector<uint32_t> unit_base(nterms + 1);
        std::vector<uint64_t> out_base(nterms + 1), host_base(nterms + 1);
        uint64_t              units{0}, posts{0}, padded{0};
        for (uint32_t i = 0; i < nterms; ++i) {
                if (term_ids[i] >= c->nterms)
                        return fail(c, TRN_ERR_ARG, "term id out of range");
                const auto &t = c->h_terms[term_ids[i]];
                unit_base[i]  = uint32_t(units);
                out_base[i]   = padded; // device rows start on a 128-entry boundary (16-byte vector stores)
                host_base[i]  = posts;
                units += (legacyDecode && c->pc.codec == TRN_CODEC_LUCENE) ? t.nblocks : (t.nblocks + 31) / 32;
                posts += t.documents;
                padded += (uint64_t(t.documents) + 127) / 128 * 128;
                if (units >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, "too many decode units");
        }
        unit_base[nterms] = uint32_t(units);
        out_base[nterms]  = padded;
        host_base[nterms] = posts;
        if (!legacyDecode) { // unit descriptors of the streaming kernels
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
        CK(c->d_dec_a.ensure(nterms * 4));
        CK(c->d_dec_b.ensure((nterms + 1) * 4));
        CK(c->d_dec_c.ensure((nterms + 1) * 8));
        CK(c->d_dec_sums.ensure(size_t(nterms) * 16));
        if (materialise) {
                CK(c->d_dec_docids.ensure(std::max<size_t>(16, padded * 4)));
                CK(c->d_dec_freqs.ensure(std::max<size_t>(16, padded * 4)));
        }
        CK(cudaMemcpyAsync(c->d_dec_a.p, term_ids, nterms * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->d_dec_b.p, unit_base.data(), (nterms + 1) * 4, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemcpyAsync(c->d_dec_c.p, out_base.data(), (nterms + 1) * 8, cudaMemcpyHostToDevice, c->stream));
        CK(cudaMemsetAsync(c->d_dec_sums.p, 0, size_t(nterms) * 16, c->stream));
        CK(cudaEventRecord(c->ev0, c->stream));
        if (units) {
                const int grid = int(std::min<uint64_t>(uint64_t(c->num_sms) * 8, (units + 3) / 4));
                // GOOGLE: the materialising variant uses the single-pass kernel with 16-byte vector stores (k_decode_google); the fused
                // checksum-only variant is faster with the span-staged kernel (scripts/microbench_decode.py compares the two)
                const bool forceNew = decodeKernel == "single-pass";
                if (!legacyDecode)
                        CK(launch_decode_stream(dev_index(c), c->d_dec_units.as<DecUnit>(), c->d_dec_c.as<uint64_t>(), uint32_t(units),
                                                materialise ? c->d_dec_docids.as<uint32_t>() : nullptr, materialise ? c->d_dec_freqs.as<uint32_t>() : nullptr,
                                                c->d_dec_sums.as<unsigned long long>(), c->num_sms, c->stream));
                else if (c->pc.codec == TRN_CODEC_GOOGLE && (materialise || forceNew))
                        CK(launch_decode_google(dev_index(c), c->d_dec_a.as<uint32_t>(), c->d_dec_b.as<uint32_t>(), c->d_dec_c.as<uint64_t>(), nterms,
                                                uint32_t(units), materialise ? c->d_dec_docids.as<uint32_t>() : nullptr,
                                                materialise ? c->d_dec_freqs.as<uint32_t>() : nullptr, c->d_dec_sums.as<unsigned long long>(), grid, c->stream));
                else
                        CK(launch_decode_terms(dev_index(c), c->d_dec_a.as<uint32_t>(), c->d_dec_b.as<uint32_t>(), c->d_dec_c.as<uint64_t>(), nterms,
                                               uint32_t(units), materialise ? c->d_dec_docids.as<uint32_t>() : nullptr,
                                               materialise ? c->d_dec_freqs.as<uint32_t>() : nullptr, c->d_dec_sums.as<unsigned long long>(), grid, c->stream));
        }
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
