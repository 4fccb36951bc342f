// trn_ctx: the device-resident index source + batch executor behind the C ABI (include/trinity_b200.h).
// Host responsibilities mirror the host side of the reference's exec path:
//   * upload == AccessProxy construction + Decoder::init for every term (google_codec.cpp:936-983, lucene_codec.cpp:877-932)
//   * plan compile == queryexec_ctx::build_iterator + build_span (exec.cpp:253-505): operator tree -> per-tile step program,
//     including the IteratorScorer combination rules of docset_iterators_scorers.cpp:8-242 (which leaves contribute to a
//     document's score is structural; see compile_node()).
// There is NO CPU execution fallback: every docset/score operation runs in kernels.cu.
#include "../../include/trinity_b200.h"
#include "codecs.h"
#include "device_types.h"
#include "hitcursor.h"
#include "chunkplan.h"
#include "kernels.h"
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
        int                  codec{0};
        int                  cand_cost{900}; // TRN_CAND_COST: modelled warp-instructions per 32 candidates of the candidate-driven conjunction (0 = never use it)
        uint32_t             block_docs{32}; // documents per full block of the uploaded index (GOOGLE 32 unless built for the decode sweep; LUCENE 128)
        uint32_t             min_docid{1}; // smallest docID any term holds (a docID-range shard does not start at 1)
        uint32_t             nterms{0}, max_docid{0}, tile_shift{13}, ntiles{0}; // tile_shift: directory granularity == scored tile (8192 docs, the reference's window docset_spans.h:74)
        uint32_t             docs_shift{14}; // docID tile (log2) of the warp-per-tile DocumentsOnly kernel
        bool                 tree_masks{false}; // TRN_TREE_MASKS=1: flat-tree queries decode their frequent leaves in a masked second pass (flat_tree_masks). It
                                                // halves the DRAM bytes, but the needed blocks of a tile fill a fraction of a 32-lane group, so the warp-instruction
                                                // count does not drop and the benchmark's trees ran slower with it. Off by default. (Not a matter of WHICH leaves
                                                // are admitted — TRN_TREE_MASK_NEED does not recover it: a few masked queries raise the launch-wide slot count and
                                                // take resident warps from every query.)
        uint32_t             tree_shift{13}; // TRN_TREE_SHIFT: docID tile (log2) of the flat-tree launch of k_exec_docs (0 = flat-tree path off)
        uint32_t             run_tiles{128};  // TRN_RUN_TILES: consecutive tiles per work item of the flat scored kernel (top-k state lives across a run)
        int                  flat_threads{320}; // TRN_SF_THREADS: CTA size of k_score_flat (256/320/384: two CTAs per SM; 512/640: one)
        uint32_t             scored_shift{13};  // TRN_SCORED_SHIFT: log2 of k_score_flat's tile (13 = the reference's window, 14)
        int                  flat_scored{1}; // TRN_FLAT_SCORED=0: every scored query through the general step-program kernel (A/B switch)
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

// flat_tree_masks: a leaf is decoded in the masked pass when at most this share of its blocks is expected to survive its mask (TRN_TREE_MASK_NEED)
static double g_tree_mask_need = 0.6;

static int fail(trn_ctx *c, int code, const std::string &m) {
        c->err = m;
        return code;
}

// =================================================================================================== plan compiler
namespace {
struct Range {
        uint32_t lo{1}, hi{0}; // inclusive docIDs; empty when lo > hi
        bool     empty() const {
                return lo > hi;
        }
};

// every node has at most one parent: a plan is a TREE (a node shared by several parents would make the recursive passes — cost, range,
// bound, truth tables — revisit it once per path, exponentially often in a hostile plan)
static bool plan_is_tree(const trn_qnode *n, uint32_t nn, uint32_t root) {
        std::vector<uint8_t> seen(nn, 0);
        if (root < nn)
                seen[root] = 1;
        for (uint32_t i = 0; i < nn; ++i) {
                if (n[i].kind == TRN_NODE_TERM)
                        continue;
                for (uint32_t k = 0; k < n[i].nchildren; ++k) {
                        const uint32_t c = uint32_t(n[i].first_child) + k;
                        if (c >= nn || seen[c])
                                return false;
                        seen[c] = 1;
                }
        }
        return true;
}

// children follow their parents in the node array (checked by validate()), so one forward pass yields every node's depth; the
// compiler and the truth-table builder recurse once per level
static bool plan_depth_ok(const trn_qnode *n, uint32_t nn) {
        std::vector<uint8_t> depth(nn, 0);
        for (uint32_t i = 0; i < nn; ++i) {
                if (n[i].kind == TRN_NODE_TERM)
                        continue;
                if (depth[i] >= 64)
                        return false;
                for (uint32_t k = 0; k < n[i].nchildren; ++k) {
                        const uint32_t c = uint32_t(n[i].first_child) + k;
                        if (c > i && c < nn)
                                depth[c] = uint8_t(std::max<int>(depth[c], depth[i] + 1));
                }
        }
        return true;
}

struct Compiler {
        const trn_qnode *           n;
        uint32_t                    nn;
        const std::vector<DevTerm> &terms;
        bool                        scored;
        uint32_t                    root;
        std::vector<DevStep> &      steps;
        uint32_t                    next_slot{0};
        uint64_t                    postings{0}, bytes{0};
        struct Deferred {
                uint32_t              term;
                double                idf;
                std::vector<uint8_t> cond;
                int                   phrase{-1}; // >= 0: node index of a phrase (its position check is repeated under the condition's mask)
        };
        std::vector<Deferred> deferred;
        std::string           err;
        bool                  reference_quirks{true};
        bool                  unsupported{false};
        bool                  allow_phrase{false}; // the caller's kernels execute OP_PHRASE (GOOGLE codec: inline hits)
        bool                  has_phrase{false};
        std::vector<uint32_t> leaf_nodes;          // node index of every OP_LEAF step, in program order (flat_tree_masks)

        Compiler(const trn_qnode *nodes, uint32_t cnt, const std::vector<DevTerm> &t, bool sc, uint32_t r, std::vector<DevStep> &s)
            : n{nodes}, nn{cnt}, terms{t}, scored{sc}, root{r}, steps{s} {
        }

        // Slots: in DocumentsOnly plans a child's bitmap is dead once it has been combined into its parent, so its slot is handed out
        // again (scored plans keep every slot: the deferred scoring pass reads branch bitmaps at the end).  Fewer live slots = less
        // shared memory per worker = more resident warps (with one slot per node the 8-term trees left few warps resident per SM).
        std::vector<uint32_t> free_slots;
        int alloc_slot() {
                if (!scored && !free_slots.empty()) {
                        const auto it = std::min_element(free_slots.begin(), free_slots.end());
                        const int  v  = int(*it);
                        free_slots.erase(it);
                        return v;
                }
                if (next_slot >= 14) {
                        err = "query needs more than 14 docset slots";
                        return -1;
                }
                return int(next_slot++);
        }
        void release_slot(uint32_t s) {
                if (!scored)
                        free_slots.push_back(s);
        }

        bool is_leaf(uint32_t i) const {
                return n[i].kind == TRN_NODE_TERM;
        }
        bool is_phrase(uint32_t i) const {
                return n[i].kind == TRN_NODE_PHRASE;
        }
        // the conjunction of a phrase's distinct terms into slot `tmp` (rarest first), then the position check in place (phrase.cuh)
        void phrase_steps(uint32_t i, uint32_t tmp, bool score) {
                const auto &          X = n[i];
                std::vector<uint32_t> t(X.nchildren);
                double                idfsum{0};
                bool                  anyEmpty{false};
                for (uint32_t j = 0; j < X.nchildren; ++j) {
                        t[j] = n[X.first_child + j].term;
                        idfsum += n[X.first_child + j].weight;
                        anyEmpty |= t[j] == kEmptyTerm || terms[t[j]].documents == 0;
                }
                if (anyEmpty) { // a phrase with an unknown term matches nothing
                        push(OP_CLEAR, 0, tmp, 0, 0, 0, 0);
                        return;
                }
                std::vector<uint32_t> distinct(t);
                std::sort(distinct.begin(), distinct.end());
                distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
                std::stable_sort(distinct.begin(), distinct.end(), [&](uint32_t a, uint32_t b) { return terms[a].documents < terms[b].documents; });
                bool first{true};
                for (auto term : distinct) {
                        postings += terms[term].documents;
                        bytes += terms[term].chunk_len;
                        push(OP_LEAF, first ? M_SET : M_AND, tmp, 0, 0, term, 0);
                        first = false;
                }
                push(OP_PHRASE, uint8_t(X.nchildren), tmp, 0, score ? F_SCORE : 0, 0, idfsum);
                for (uint32_t j = 0; j < X.nchildren; j += 4) { // four term ids per operand step, in phrase order
                        DevStep a;
                        std::memset(&a, 0, sizeof(a));
                        a.op   = OP_ARG;
                        a.term = t[j];
                        a.pad2 = j + 1 < X.nchildren ? t[j + 1] : 0u;
                        const uint64_t hi = uint64_t(j + 2 < X.nchildren ? t[j + 2] : 0u) | (uint64_t(j + 3 < X.nchildren ? t[j + 3] : 0u) << 32);
                        std::memcpy(&a.idf, &hi, 8);
                        steps.push_back(a);
                }
        }
        // a phrase operand combined into dst with `mode` (== leaf() for a term); scores score(matchCnt, sum idf) where it holds
        bool phrase_leaf(uint32_t i, uint8_t mode, uint32_t dst, bool scoring, const std::vector<uint8_t> &cond, uint8_t extraFlags) {
                const bool wantScore = scored && scoring;
                if (mode == M_NONE && !wantScore)
                        return true; // nothing to do in this pass
                const bool immediate = wantScore && cond.empty();
                if (wantScore && !immediate)
                        deferred.push_back({0, 0.0, cond, int(i)});
                if (mode == M_NONE && !immediate)
                        return true; // the deferred pass does it all
                const int tmp = alloc_slot();
                if (tmp < 0)
                        return false;
                phrase_steps(i, uint32_t(tmp), immediate);
                if (mode != M_NONE)
                        push(OP_SLOT, mode, dst, uint32_t(tmp), extraFlags, 0, 0);
                release_slot(uint32_t(tmp));
                return true;
        }
        uint32_t df(uint32_t i) const {
                const auto t = n[i].term;
                return t == kEmptyTerm ? 0u : terms[t].documents;
        }
        void push(uint8_t op, uint8_t mode, uint32_t dst, uint32_t src, uint8_t flags, uint32_t term, double idf) {
                DevStep s;
                std::memset(&s, 0, sizeof(s));
                s.op    = op;
                s.mode  = mode;
                s.dst   = uint8_t(dst);
                s.src   = uint8_t(src);
                s.flags = flags;
                s.term  = term;
                s.idf   = idf;
                steps.push_back(s);
        }
        void account(uint32_t i) {
                const auto t = n[i].term;
                if (t != kEmptyTerm) {
                        postings += terms[t].documents;
                        bytes += terms[t].chunk_len;
                }
        }
        // leaf combined into dst with `mode`; scoring per the structural rules
        void leaf(uint32_t i, uint8_t mode, uint32_t dst, bool scoring, const std::vector<uint8_t> &cond, uint8_t extraFlags) {
                account(i);
                uint8_t flags = extraFlags;
                if (scored && scoring) {
                        if (cond.empty())
                                flags |= F_SCORE;
                        else
                                deferred.push_back({n[i].term, n[i].weight, cond});
                }
                if (mode == M_NONE && !(flags & F_SCORE))
                        return; // nothing to do in this pass
                leaf_nodes.push_back(i);
                push(OP_LEAF, mode, dst, 0, flags, n[i].term, n[i].weight);
        }

        // compiles internal node i into its own slot; returns the slot
        int node(uint32_t i, bool scoring, const std::vector<uint8_t> &cond) {
                const int sAlloc = alloc_slot();
                if (sAlloc < 0)
                        return -1;
                const uint32_t s    = uint32_t(sAlloc);
                const auto &   X    = n[i];
                const bool     isRoot = i == root;
                if (X.nchildren == 0 || uint32_t(X.first_child) + X.nchildren > nn) {
                        err = "operator node without (valid) children";
                        return -1;
                }
                std::vector<uint32_t> kids(X.nchildren);
                for (uint32_t c = 0; c < X.nchildren; ++c)
                        kids[c] = X.first_child + c;
                auto child_cond = [&](uint32_t slotOfChild) {
                        auto v = cond;
                        v.push_back(uint8_t(slotOfChild));
                        return v;
                };
                switch (X.kind) {
                        case TRN_NODE_AND: {
                                // leaves first, rarest first (== prepare_tree's df sort exec.cpp:154-170 and reorder_execnodes :216)
                                std::stable_sort(kids.begin(), kids.end(), [&](uint32_t a, uint32_t b) {
                                        const bool la = is_leaf(a), lb = is_leaf(b);
                                        if (la != lb)
                                                return la;
                                        if (la)
                                                return df(a) < df(b);
                                        return false;
                                });
                                bool first{true};
                                for (auto c : kids) {
                                        const uint8_t fl = isRoot ? F_BREAK_IF_EMPTY : 0;
                                        if (is_leaf(c))
                                                leaf(c, first ? M_SET : M_AND, s, scoring, cond, fl);
                                        else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, first ? M_SET : M_AND, s, scoring, cond, fl))
                                                        return -1;
                                        } else {
                                                const int cs = node(c, scoring, cond);
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, first ? M_SET : M_AND, s, uint32_t(cs), fl, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                        first = false;
                                }
                        } break;
                        case TRN_NODE_OR: {
                                push(OP_CLEAR, 0, s, 0, 0, 0, 0);
                                for (auto c : kids) {
                                        if (is_leaf(c))
                                                leaf(c, M_OR, s, scoring, cond, 0);
                                        else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, M_OR, s, scoring, cond, 0))
                                                        return -1;
                                        } else {
                                                // a non-leaf child of a disjunction contributes its score only for documents it matches itself
                                                // (Disjunction scorer sums children positioned on the doc, docset_iterators_scorers.cpp)
                                                const uint32_t willBe = next_slot;
                                                const int      cs     = node(c, scoring, child_cond(willBe));
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, M_OR, s, uint32_t(cs), 0, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                }
                        } break;
                        case TRN_NODE_NOT:
                        case TRN_NODE_OPTIONAL: {
                                if (X.nchildren != 2) {
                                        err = "NOT / OPTIONAL need exactly two children";
                                        return -1;
                                }
                                const uint8_t fl = isRoot ? F_BREAK_IF_EMPTY : 0;
                                if (is_leaf(kids[0]))
                                        leaf(kids[0], M_SET, s, scoring, cond, fl);
                                else if (is_phrase(kids[0])) {
                                        if (!phrase_leaf(kids[0], M_SET, s, scoring, cond, fl))
                                                return -1;
                                } else {
                                        const int cs = node(kids[0], scoring, cond);
                                        if (cs < 0)
                                                return -1;
                                        push(OP_SLOT, M_SET, s, uint32_t(cs), fl, 0, 0);
                                        release_slot(uint32_t(cs));
                                }
                                if (X.kind == TRN_NODE_NOT) {
                                        // Filter: excluded side never scores (docset_iterators_scorers.cpp Filter -> req only)
                                        if (is_leaf(kids[1]))
                                                leaf(kids[1], M_ANDNOT, s, false, cond, 0);
                                        else if (is_phrase(kids[1])) {
                                                if (!phrase_leaf(kids[1], M_ANDNOT, s, false, cond, 0))
                                                        return -1;
                                        } else {
                                                const int cs = node(kids[1], false, cond);
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, M_ANDNOT, s, uint32_t(cs), 0, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                } else if (scored && scoring) {
                                        // Optional: main drives; opt only adds its score when it is on the document
                                        if (is_leaf(kids[1]))
                                                leaf(kids[1], M_NONE, s, true, cond, 0);
                                        else if (is_phrase(kids[1])) {
                                                if (!phrase_leaf(kids[1], M_NONE, s, true, cond, 0))
                                                        return -1;
                                        } else {
                                                const uint32_t willBe = next_slot;
                                                if (node(kids[1], true, child_cond(willBe)) < 0)
                                                        return -1;
                                        }
                                } else {
                                        // docs-only: the optional side cannot change the match set, but it is still "touched" by the reference
                                        // (Optional::next advances opt lazily); we do not read it at all.
                                }
                        } break;
                        case TRN_NODE_SOME: {
                                // DisjunctionSome (docset_iterators.cpp:679-811): every child is evaluated into a bitmap of its own and added to a
                                // bit-sliced saturating counter (one bitmap per counter bit); the node matches where the counter reaches `min`.
                                // A child scores only where it matches AND the node matches (Wrapper::iterator_score sums the lead list).
                                const uint32_t m = X.term;
                                if (m == 0 || m > 15) {
                                        err = "SOME: min-should-match must be in 1..15";
                                        return -1;
                                }
                                uint32_t k = 1;
                                while (((1u << k) - 1u) < m)
                                        ++k;
                                if (next_slot + k + 1 > 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                const uint32_t p0 = next_slot;
                                next_slot += k;
                                const uint32_t t = next_slot++; // shared by the leaf children
                                for (uint32_t j = 0; j < k; ++j)
                                        push(OP_CLEAR, 0, p0 + j, 0, 0, 0, 0);
                                for (auto c : kids) {
                                        uint32_t src;
                                        if (is_leaf(c)) {
                                                leaf(c, M_SET, t, scoring, child_cond(s), 0);
                                                src = t;
                                        } else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, M_SET, t, scoring, child_cond(s), 0))
                                                        return -1;
                                                src = t;
                                        } else {
                                                auto cc = child_cond(s);
                                                cc.push_back(uint8_t(next_slot)); // the child's own slot
                                                const int cs = node(c, scoring, cc);
                                                if (cs < 0)
                                                        return -1;
                                                src = uint32_t(cs);
                                        }
                                        push(OP_COUNT_ADD, uint8_t(k), p0, src, 0, 0, 0);
                                        if (src != t)
                                                release_slot(src);
                                }
                                push(OP_COUNT_GE, uint8_t(k), s, p0, 0, m, 0);
                                for (uint32_t j = 0; j < k; ++j)
                                        release_slot(p0 + j);
                                release_slot(t);
                        } break;
                        default:
                                err = "unknown node kind";
                                return -1;
                }
                return int(s);
        }

        Range range(uint32_t i) const {
                const auto &X = n[i];
                Range       r;
                if (X.kind == TRN_NODE_TERM) {
                        if (X.term != kEmptyTerm && terms[X.term].documents) {
                                r.lo = terms[X.term].first_doc;
                                r.hi = terms[X.term].last_doc;
                        }
                        return r;
                }
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return range(X.first_child);
                const bool conj = X.kind == TRN_NODE_AND || X.kind == TRN_NODE_PHRASE; // a phrase needs all of its terms
                bool       first{true};
                for (uint32_t c = 0; c < X.nchildren; ++c) {
                        const Range cr = range(X.first_child + c);
                        if (conj) {
                                if (cr.empty())
                                        return Range{};
                                if (first)
                                        r = cr;
                                else {
                                        r.lo = std::max(r.lo, cr.lo);
                                        r.hi = std::min(r.hi, cr.hi);
                                        if (r.empty())
                                                return Range{};
                                }
                                first = false;
                        } else {
                                if (cr.empty())
                                        continue;
                                if (first)
                                        r = cr;
                                else {
                                        r.lo = std::min(r.lo, cr.lo);
                                        r.hi = std::max(r.hi, cr.hi);
                                }
                                first = false;
                        }
                }
                return r;
        }

        uint64_t bound(uint32_t i) const {
                const auto &X = n[i];
                if (X.kind == TRN_NODE_TERM)
                        return df(i);
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return bound(X.first_child);
                const bool conj = X.kind == TRN_NODE_AND || X.kind == TRN_NODE_PHRASE;
                uint64_t   b    = conj ? ~0ull : 0ull;
                for (uint32_t c = 0; c < X.nchildren; ++c) {
                        const uint64_t cb = bound(X.first_child + c);
                        b                 = conj ? std::min(b, cb) : b + cb;
                }
                return b;
        }

        bool validate() {
                if (root >= nn) {
                        err = "root out of range";
                        return false;
                }
                if (!plan_depth_ok(n, nn)) {
                        err = "query tree deeper than 64 levels";
                        return false;
                }
                for (uint32_t i = 0; i < nn; ++i) {
                        if (n[i].kind == TRN_NODE_TERM) {
                                if (n[i].term != kEmptyTerm && n[i].term >= terms.size()) {
                                        err = "term id out of range";
                                        return false;
                                }
                        } else if (n[i].kind == TRN_NODE_PHRASE) {
                                if (!allow_phrase) {
                                        err         = "phrase nodes need the positions (materialize_hits): a LUCENE source executes them once its hits.data has been uploaded (trn_upload_hits)";
                                        unsupported = true;
                                        return false;
                                }
                                if (n[i].nchildren < 2 || n[i].nchildren > 16 || n[i].first_child <= i || uint32_t(n[i].first_child) + n[i].nchildren > nn) {
                                        err = "a phrase holds 2..16 terms behind it in the node array";
                                        return false;
                                }
                                for (uint32_t k = 0; k < n[i].nchildren; ++k)
                                        if (n[n[i].first_child + k].kind != TRN_NODE_TERM) {
                                                err = "the children of a phrase are terms";
                                                return false;
                                        }
                                has_phrase = true;
                        } else if (n[i].kind > TRN_NODE_PHRASE) {
                                err = "unknown node kind";
                                return false;
                        } else {
                                // children must come after their parent (guarantees an acyclic tree)
                                if (n[i].nchildren == 0 || n[i].first_child <= i || uint32_t(n[i].first_child) + n[i].nchildren > nn) {
                                        err = "children must follow their parent in the node array";
                                        return false;
                                }
                        }
                }
                if (!plan_is_tree(n, nn, root)) {
                        err = "a node is referenced by more than one parent (a plan is a tree)";
                        return false;
                }
                return true;
        }

        // == DocsSetIterators::cost() (docset_iterators.cpp:10-64); a conjunction's cost is its lead's, which the reference's
        // reordering passes make the cheapest operand
        uint64_t cost(uint32_t i) const {
                const auto &X = n[i];
                if (X.kind == TRN_NODE_TERM)
                        return df(i);
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return cost(X.first_child);
                if (X.kind == TRN_NODE_PHRASE) // docset_iterators.cpp:50-55: cost(its[0]) + UINT32_MAX + UINT16_MAX * size
                        return cost(X.first_child) + 0xffffffffull + 0xffffull * X.nchildren;
                if (X.kind == TRN_NODE_SOME) { // DisjunctionSome::cost_: the (size - min + 1) cheapest children (docset_iterators.cpp:733-742)
                        std::vector<uint64_t> cs;
                        for (uint32_t k = 0; k < X.nchildren; ++k)
                                cs.push_back(cost(X.first_child + k));
                        std::sort(cs.begin(), cs.end());
                        const uint32_t keep = X.nchildren >= X.term ? X.nchildren - X.term + 1u : 0u;
                        uint64_t       c{0};
                        for (uint32_t k = 0; k < keep && k < cs.size(); ++k)
                                c += cs[k];
                        return c;
                }
                uint64_t c = X.kind == TRN_NODE_AND ? ~0ull : 0ull;
                for (uint32_t k = 0; k < X.nchildren; ++k) {
                        const uint64_t cc = cost(X.first_child + k);
                        c                 = X.kind == TRN_NODE_AND ? std::min(c, cc) : c + cc;
                }
                return c;
        }

        // REFERENCE QUIRK, mirrored for drop-in parity: build_span() (exec.cpp:488-501) turns a root Filter whose excluded side is not
        // costlier than its required side into FilteredDocsSetSpan(build_span(req), excl).  When req is a disjunction the inner span is
        // DocsSetSpanForDisjunctions[WithThreshold], whose process() ignores its `min` argument (docset_spans.cpp:98-111,681-694): the
        // excluded documents the outer span stepped over are emitted by the next call anyway, so the exclusion has no effect and the
        // reference returns the plain disjunction.  The same holds through a chain of such root filters.
        void apply_reference_root_filter_quirk() {
                uint32_t cur = root;
                bool     traversed{false};
                while (n[cur].kind == TRN_NODE_NOT && n[cur].nchildren == 2 && cost(n[cur].first_child + 1u) <= cost(n[cur].first_child)) {
                        cur       = n[cur].first_child;
                        traversed = true;
                }
                if (traversed && n[cur].kind == TRN_NODE_OR)
                        root = cur;
        }

        // returns root slot or -1
        int run() {
                if (!validate())
                        return -1;
                if (reference_quirks)
                        apply_reference_root_filter_quirk();
                int rs;
                if (is_leaf(root)) {
                        rs = int(next_slot++);
                        leaf(root, M_SET, uint32_t(rs), true, {}, 0);
                } else if (is_phrase(root)) {
                        rs = int(next_slot++);
                        if (!phrase_leaf(root, M_SET, uint32_t(rs), true, {}, 0))
                                return -1;
                } else
                        rs = node(root, true, {});
                if (rs < 0)
                        return -1;
                // second pass for leaves whose contribution is conditional on a disjunction branch matching
                for (auto &d : deferred) {
                        uint32_t mask = d.cond[0];
                        if (d.cond.size() > 1) {
                                if (next_slot >= 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                mask = next_slot++;
                                push(OP_SLOT, M_SET, mask, d.cond[0], 0, 0, 0);
                                for (size_t j = 1; j < d.cond.size(); ++j)
                                        push(OP_SLOT, M_AND, mask, d.cond[j], 0, 0, 0);
                        }
                        if (d.phrase >= 0) { // the phrase again, restricted to the condition's documents, scoring this time
                                if (next_slot >= 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                const uint32_t tmp = next_slot++;
                                // (phrase_steps starts with SET/CLEAR into tmp; the mask narrows the candidates before the position check)
                                const size_t at = steps.size();
                                phrase_steps(uint32_t(d.phrase), tmp, true);
                                // insert [SLOT AND tmp, mask] in front of the OP_PHRASE step
                                for (size_t z = at; z < steps.size(); ++z)
                                        if (steps[z].op == OP_PHRASE) {
                                                DevStep a;
                                                std::memset(&a, 0, sizeof(a));
                                                a.op   = OP_SLOT;
                                                a.mode = M_AND;
                                                a.dst  = uint8_t(tmp);
                                                a.src  = uint8_t(mask);
                                                steps.insert(steps.begin() + z, a);
                                                break;
                                        }
                                continue;
                        }
                        push(OP_LEAFSCORE, M_NONE, 0, mask, 0, d.term, d.idf);
                }
                return rs;
        }
};
} // namespace

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
        if (const char *e = getenv("TRN_TILE_SHIFT")) { // directory granularity == tile of the scored kernel (experiments)
                const int v = atoi(e);
                if (v >= 12 && v <= 14)
                        c->tile_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_CAND_COST"))
                c->cand_cost = std::max(0, atoi(e));
        if (const char *e = getenv("TRN_DOCS_SHIFT")) {
                const int v = atoi(e);
                if (v >= 13 && v <= 17)
                        c->docs_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_TREE_SHIFT")) {
                const int v = atoi(e);
                if (v == 0 || (v >= 10 && v <= 14))
                        c->tree_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_TREE_MASKS"))
                c->tree_masks = atoi(e) != 0;
        if (const char *e = getenv("TRN_TREE_MASK_NEED")) {
                const double v = atof(e);
                if (v > 0.0 && v <= 1.0)
                        g_tree_mask_need = v;
        }
        if (const char *e = getenv("TRN_RUN_TILES")) {
                const int v = atoi(e);
                if (v >= 1 && v <= 4096)
                        c->run_tiles = uint32_t(v);
        }
        if (const char *e = getenv("TRN_FLAT_SCORED"))
                c->flat_scored = atoi(e) != 0;
        if (const char *e = getenv("TRN_SF_THREADS"))
                c->flat_threads = atoi(e);
        if (const char *e = getenv("TRN_SCORED_SHIFT")) {
                const int v = atoi(e);
                if (v == 13 || v == 14)
                        c->scored_shift = uint32_t(v);
        }
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
        BlockDirectory dir;
        try {
                std::vector<term_index_ctx> t(nterms);
                for (uint32_t i = 0; i < nterms; ++i) {
                        t[i].documents = terms[i].documents;
                        t[i].offset    = terms[i].chunk_off;
                        t[i].size      = terms[i].chunk_len;
                }
                const int threads = int(std::max(1u, std::min(64u, std::thread::hardware_concurrency())));
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, t.data(), nterms, threads, dir);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_index: out of host memory while building the block directory");
        } catch (const std::exception &e) {
                return fail(c, TRN_ERR_FORMAT, e.what());
        }
        if (max_docid == 0) // not recorded (e.g. a segment directory): the largest docID any postings list holds
                for (uint32_t i = 0; i < nterms; ++i)
                        if (dir.terms[i].nblocks)
                                max_docid = std::max(max_docid, dir.terms[i].last_doc);
        c->codec      = codec;
        c->block_docs = dir.block_docs;
        c->nterms     = nterms;
        c->max_docid  = max_docid;
        const uint32_t W = 1u << c->tile_shift;
        c->ntiles     = uint32_t((uint64_t(max_docid) + 1 + W - 1) >> c->tile_shift);
        try {
                c->h_terms.resize(nterms);
        } catch (const std::bad_alloc &) {
                return fail(c, TRN_ERR_CAPACITY, "trn_upload_index: out of host memory");
        }
        c->have_index     = false; // until the new index is completely in place
        c->min_docid      = 0xffffffffu;
        c->total_blocks   = 0;
        c->total_postings = 0;
        for (uint32_t i = 0; i < nterms; ++i) {
                auto &d     = c->h_terms[i];
                d.documents = dir.terms[i].documents;
                d.dir_begin = dir.terms[i].dir_begin;
                d.nblocks   = dir.terms[i].nblocks;
                d.first_doc = dir.terms[i].first_doc;
                d.last_doc  = dir.terms[i].last_doc;
                d.chunk_len = terms[i].chunk_len;
                d.tf_begin  = dir.terms[i].tf_begin;
                d.tf_base   = dir.terms[i].tf_base;
                d.tf_shift  = dir.terms[i].tf_shift;
                c->total_blocks += d.nblocks;
                c->total_postings += d.documents;
                if (d.nblocks)
                        c->min_docid = std::min(c->min_docid, d.first_doc);
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
        if (c->codec != TRN_CODEC_LUCENE)
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
        const uint64_t        span  = ((uint64_t(c->max_docid) >> 17) + 2) << 17;
        std::vector<uint32_t> words(span / 32, 0u);
        for (uint64_t i = 0; i < n; ++i) {
                if (docids[i] == 0)
                        return fail(c, TRN_ERR_ARG, "masked docID 0 is not a document");
                if (docids[i] > c->max_docid)
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
        o->codec           = c->codec;
        o->nterms          = c->nterms;
        o->max_docid       = c->max_docid;
        o->tile_docs       = 1u << c->tile_shift;
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
        ix.tile_shift = c->tile_shift;
        ix.max_docid  = c->max_docid;
        ix.block_docs = c->block_docs;
        ix.codec      = c->codec;
        ix.hits       = c->have_hits ? c->d_hits.as<uint8_t>() : nullptr;
        ix.hit_base   = c->have_hits ? c->d_hit_base.as<uint32_t>() : nullptr;
        ix.hblk_off   = c->have_hits ? c->d_hblk_off.as<uint32_t>() : nullptr;
        ix.hit_term   = c->have_hits ? c->d_hit_term.as<HitTerm>() : nullptr;
        return ix;
}

// Truth vector of a query subtree over its (<= 8) distinct terms: bit `a` (0..255) = value of the node when exactly the terms whose
// bit is set in `a` are present (bit j of `a` = term tv[j]).  Bitwise evaluation: one 256-bit operation per node.
struct TruthVec {
        uint64_t w[4];
};
static TruthVec truth_vector(const trn_qnode *nodes, uint32_t i, const uint32_t *tv, uint32_t n) {
        static const uint64_t kPat[6] = {0xaaaaaaaaaaaaaaaaull, 0xccccccccccccccccull, 0xf0f0f0f0f0f0f0f0ull, 0xff00ff00ff00ff00ull, 0xffff0000ffff0000ull, 0xffffffff00000000ull};
        const auto &X = nodes[i];
        TruthVec    v{{0, 0, 0, 0}};
        if (X.kind == TRN_NODE_TERM) {
                for (uint32_t j = 0; j < n; ++j)
                        if (tv[j] == X.term) {
                                for (int q = 0; q < 4; ++q)
                                        v.w[q] = j < 6 ? kPat[j] : (j == 6 ? ((q & 1) ? ~0ull : 0ull) : ((q & 2) ? ~0ull : 0ull));
                                break;
                        }
                return v;
        }
        const uint32_t f = X.first_child;
        if (X.kind == TRN_NODE_SOME) {
                const uint32_t        nk = X.nchildren; // all of them (<= 255)
                std::vector<TruthVec> kids(nk);
                for (uint32_t k = 0; k < nk; ++k)
                        kids[k] = truth_vector(nodes, f + k, tv, n);
                for (uint32_t a = 0; a < 256; ++a) {
                        uint32_t cnt{0};
                        for (uint32_t k = 0; k < nk; ++k)
                                cnt += uint32_t((kids[k].w[a >> 6] >> (a & 63u)) & 1ull);
                        if (cnt >= X.term)
                                v.w[a >> 6] |= 1ull << (a & 63u);
                }
                return v;
        }
        v = truth_vector(nodes, f, tv, n);
        for (uint32_t k = 1; k < X.nchildren; ++k) {
                const TruthVec w = truth_vector(nodes, f + k, tv, n);
                for (int q = 0; q < 4; ++q) {
                        if (X.kind == TRN_NODE_AND) v.w[q] &= w.w[q];
                        else if (X.kind == TRN_NODE_OR) v.w[q] |= w.w[q];
                        else if (X.kind == TRN_NODE_NOT) v.w[q] &= ~w.w[q];
                        // OPTIONAL: the optional side never changes the match set
                }
        }
        return v;
}

extern "C" int trn_query_truth_table(const trn_qnode *nodes, uint32_t nnodes, uint32_t root, uint32_t *terms, uint32_t *nterms, uint32_t *table, uint32_t *necessary) {
        if (!nodes || !nnodes || root >= nnodes || !terms || !nterms || !table || !necessary)
                return TRN_ERR_ARG;
        for (uint32_t i = 0; i < nnodes; ++i) // same structural rules as the plan compiler: children behind their parent, bounded depth
                if (nodes[i].kind != TRN_NODE_TERM && (nodes[i].nchildren == 0 || nodes[i].first_child <= i || uint32_t(nodes[i].first_child) + nodes[i].nchildren > nnodes))
                        return TRN_ERR_ARG;
        if (!plan_depth_ok(nodes, nnodes) || !plan_is_tree(nodes, nnodes, root))
                return TRN_ERR_ARG;
        uint32_t n{0}, stack[64], sp{0};
        stack[sp++] = root;
        while (sp) {
                const auto &X = nodes[stack[--sp]];
                if (X.kind == TRN_NODE_TERM) {
                        if (X.term == kEmptyTerm)
                                continue;
                        bool seen{false};
                        for (uint32_t j = 0; j < n; ++j)
                                seen |= terms[j] == X.term;
                        if (!seen) {
                                if (n == 8)
                                        return TRN_ERR_ARG;
                                terms[n++] = X.term;
                        }
                } else {
                        if (X.kind == TRN_NODE_PHRASE)
                                return TRN_ERR_UNSUPPORTED;
                        if (X.kind > TRN_NODE_SOME || X.nchildren == 0 || uint32_t(X.first_child) + X.nchildren > nnodes || sp + X.nchildren > 64)
                                return TRN_ERR_ARG;
                        for (uint32_t k = 0; k < X.nchildren; ++k)
                                stack[sp++] = X.first_child + k;
                }
        }
        const TruthVec v = truth_vector(nodes, root, terms, n);
        uint32_t       nec{n ? (1u << n) - 1u : 0u};
        for (uint32_t w = 0; w < 8; ++w)
                table[w] = 0;
        for (uint32_t a = 0; a < (1u << n); ++a)
                if ((v.w[a >> 6] >> (a & 63u)) & 1ull) {
                        table[a >> 5] |= 1u << (a & 31u);
                        nec &= a;
                }
        *nterms    = n;
        *necessary = nec;
        return TRN_OK;
}

// Flat-tree form of a DocumentsOnly step program (k_exec_docs, exec_docs_flat.cuh): every leaf gets a bitmap of its own (slots 0 .. nl-1,
// announced by one [OP_LEAF M_NONE dst = leaf slot] marker each, at the front of the program) that ONE flat (leaf, block) pass over the tile
// fills; the rest of the program becomes slot operations on them, the compiler's own slots moved behind the leaf bitmaps.
// Returns the number of leaves (0: the program stays as it is).
// Leaf bitmaps are numbered by descending block count: the (leaf, block) list of a tile is then ordered from the frequent terms (blocks
// of 1-byte deltas, four codes per decoder step) to the rare ones (2-byte deltas, blocks that straddle the tile), so that the 32 lanes
// of a group mostly walk blocks of the same kind — a rare term's lane among frequent ones kept the whole warp in the loop for its 16-31
// slow steps (those ran at a few of 32 lanes and were as many instructions as the fast ones).
// Afterwards the copies are coalesced (flat_tree_coalesce): `SET d <- s` where s is not read again becomes a renaming of d, so a chain
// like SET t <- leaf; AND t, leaf2; OR acc, t runs in the leaf's own bitmap: fewer operations per tile and — what matters more — fewer
// bitmaps per warp (13 -> 8 for the 8-term trees of the benchmark), i.e. more resident warps.
// rootSlot: in = the compiler's root slot, out = the slot that holds the root docset; slotsInUse: out.
static void     flat_tree_coalesce(std::vector<DevStep> &steps, size_t opsBegin, uint32_t nl, uint32_t &rootSlot, uint32_t &slotsInUse);
static uint32_t flat_tree_transform(std::vector<DevStep> &steps, size_t begin, uint32_t next_slot, const std::vector<DevTerm> &terms, std::vector<uint32_t> *leafNodes,
                                    uint32_t &rootSlot, uint32_t &slotsInUse) {
        uint32_t nl{0};
        for (size_t i = begin; i < steps.size(); ++i)
                nl += steps[i].op == OP_LEAF && steps[i].mode != M_NONE;
        uint32_t nops{nl}; // slot operations of the transformed program: one per decoding leaf + every non-leaf step
        for (size_t i = begin; i < steps.size(); ++i)
                nops += steps[i].op != OP_LEAF;
        if (nl < 2 || nl > 16 || nl + next_slot > 30 || nops > 32)
                return 0; // (the kernel keeps leaves and slot operations in lane registers: <= 16 leaves, <= 32 operations, slots < 32)
        for (size_t i = begin; i < steps.size(); ++i)
                if (steps[i].op == OP_COUNT_GE && steps[i].term > 15u)
                        return 0;
        const std::vector<DevStep> prog(steps.begin() + begin, steps.end());
        steps.resize(begin);
        std::vector<DevStep> leaves;
        for (const auto &st : prog)
                if (st.op == OP_LEAF && st.mode != M_NONE)
                        leaves.push_back(st);
        std::vector<uint32_t> order(nl), slotOf(nl); // order[k]: program leaf held by bitmap k; slotOf: its inverse
        for (uint32_t j = 0; j < nl; ++j)
                order[j] = j;
        auto blocksOf = [&](uint32_t j) { return leaves[j].term == kEmptyTerm ? 0u : terms[leaves[j].term].nblocks; };
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return blocksOf(a) > blocksOf(b); });
        for (uint32_t k = 0; k < nl; ++k) {
                slotOf[order[k]] = k;
                DevStep L        = leaves[order[k]]; // decode marker: term -> leaf bitmap k
                L.mode           = M_NONE;
                L.dst            = uint8_t(k);
                L.src            = 0;
                L.flags          = 0;
                steps.push_back(L);
        }
        if (leafNodes && leafNodes->size() == nl) {
                const std::vector<uint32_t> was(*leafNodes);
                for (uint32_t k = 0; k < nl; ++k)
                        (*leafNodes)[k] = was[order[k]];
        }
        uint32_t li{0};
        for (auto st : prog) {
                if (st.op == OP_LEAF) {
                        if (st.mode == M_NONE)
                                continue; // nothing to do in DocumentsOnly mode
                        DevStep S;
                        std::memset(&S, 0, sizeof(S));
                        S.op    = OP_SLOT;
                        S.mode  = st.mode;
                        S.dst   = uint8_t(st.dst + nl);
                        S.src   = uint8_t(slotOf[li++]);
                        S.flags = st.flags;
                        steps.push_back(S);
                        continue;
                }
                st.dst = uint8_t(st.dst + nl); // compiler slots live behind the leaf bitmaps
                if (st.op == OP_SLOT || st.op == OP_COUNT_ADD || st.op == OP_COUNT_GE)
                        st.src = uint8_t(st.src + nl);
                steps.push_back(st);
        }
        rootSlot += nl;
        slotsInUse = nl + next_slot;
        flat_tree_coalesce(steps, begin + nl, nl, rootSlot, slotsInUse);
        return nl;
}

static void flat_tree_coalesce(std::vector<DevStep> &steps, size_t opsBegin, uint32_t nl, uint32_t &rootSlot, uint32_t &slotsInUse) {
        std::vector<DevStep> ops(steps.begin() + std::ptrdiff_t(opsBegin), steps.end());
        for (const auto &o : ops)
                if (o.op != OP_SLOT && o.op != OP_CLEAR)
                        return; // (counter planes address slot RANGES: left alone)
        auto reads = [](const DevStep &o, uint32_t x) { // does o read slot x?
                if (o.op != OP_SLOT)
                        return false;
                if (o.mode == M_NONE)
                        return o.dst == x; // emptiness test only
                return o.src == x || (o.mode != M_SET && o.dst == x);
        };
        auto overwrites = [](const DevStep &o, uint32_t x) { return o.dst == x && (o.op == OP_CLEAR || (o.op == OP_SLOT && o.mode == M_SET)); };
        // x is dead behind operation i: nothing reads it before it is overwritten, and it is not the root
        auto dead = [&](size_t i, uint32_t x) {
                for (size_t j = i + 1; j < ops.size(); ++j) {
                        if (reads(ops[j], x))
                                return false;
                        if (overwrites(ops[j], x))
                                return true;
                }
                return x != rootSlot;
        };
        // CLEAR d ... OR d, x (nothing touching d in between)  ==  SET d <- x
        std::vector<uint8_t> drop(ops.size(), 0);
        for (size_t i = 0; i < ops.size(); ++i) {
                if (ops[i].op != OP_CLEAR)
                        continue;
                const uint32_t d = ops[i].dst;
                for (size_t j = i + 1; j < ops.size(); ++j) {
                        const bool touches = ops[j].dst == d || (ops[j].op == OP_SLOT && ops[j].src == d);
                        if (!touches)
                                continue;
                        if (ops[j].op == OP_SLOT && ops[j].mode == M_OR && ops[j].dst == d && ops[j].src != d) {
                                ops[j].mode = M_SET;
                                drop[i]     = 1;
                        }
                        break;
                }
        }
        // forward renaming: ren[name] = the physical slot that holds it, holder[slot] = the name it holds (the compiler hands slot numbers
        // out again, so a name that is overwritten must not land in a slot that meanwhile carries another live name)
        uint32_t ren[32], holder[32];
        for (uint32_t i = 0; i < 32; ++i)
                ren[i] = holder[i] = i;
        auto deadFrom = [&](size_t i, uint32_t x) { // like dead(), operation i included
                if (x >= 32u)
                        return true;
                if (i < ops.size() && reads(ops[i], x))
                        return false;
                if (i < ops.size() && overwrites(ops[i], x))
                        return true;
                return dead(i, x);
        };
        std::vector<DevStep> out;
        for (size_t i = 0; i < ops.size(); ++i) {
                if (drop[i])
                        continue;
                DevStep o = ops[i];
                if (o.op == OP_SLOT && o.mode == M_SET && o.src != o.dst && dead(i, o.src)) {
                        const uint32_t p = ren[o.src];
                        if (holder[ren[o.dst]] == o.dst)
                                holder[ren[o.dst]] = 0xffu;
                        ren[o.dst] = p;
                        holder[p]  = o.dst;
                        if (o.flags & F_BREAK_IF_EMPTY) { // the emptiness test stays, on the slot that now carries the name
                                o.mode = M_NONE;
                                o.dst  = uint8_t(p);
                                o.src  = uint8_t(p);
                                out.push_back(o);
                        }
                        continue;
                }
                if (o.op == OP_SLOT)
                        o.src = uint8_t(ren[o.src]);
                if (o.op == OP_CLEAR || (o.op == OP_SLOT && o.mode == M_SET)) { // a full overwrite: the name needs a slot nobody lives in
                        uint32_t p = ren[o.dst];
                        if (holder[p] != o.dst && !deadFrom(i, holder[p])) {
                                p = 0xffu;
                                for (uint32_t k = 0; k < 31u && p == 0xffu; ++k) {
                                        const uint32_t q = k + nl < 31u ? k + nl : k + nl - 31u; // compiler slots first, then leaf bitmaps already consumed
                                        if (deadFrom(i, holder[q]) && !(o.op == OP_SLOT && q == o.src))
                                                p = q;
                                }
                                if (p == 0xffu)
                                        return; // (cannot happen: the program had a slot for every live name) leave the program as it was
                        }
                        ren[o.dst] = p;
                        holder[p]  = o.dst;
                }
                o.dst = uint8_t(ren[o.dst]);
                out.push_back(o);
        }
        rootSlot = ren[rootSlot];
        // compiler slots still in use, renumbered densely behind the leaf bitmaps
        uint32_t map[32];
        uint32_t next = nl;
        for (uint32_t i = 0; i < 32; ++i)
                map[i] = i < nl ? i : 0xffu;
        auto use = [&](uint32_t x) {
                if (x >= nl && map[x] == 0xffu)
                        map[x] = next++;
        };
        for (const auto &o : out) {
                use(o.dst);
                if (o.op == OP_SLOT)
                        use(o.src);
        }
        use(rootSlot);
        for (auto &o : out) {
                o.dst = uint8_t(map[o.dst]);
                if (o.op == OP_SLOT)
                        o.src = uint8_t(map[o.src]);
        }
        rootSlot   = map[rootSlot];
        slotsInUse = next;
        steps.resize(opsBegin);
        steps.insert(steps.end(), out.begin(), out.end());
}

// Masked second decode pass of the flat-tree path.  A leaf whose blocks are short in docID terms (a frequent term) does not have to be
// decoded where the rest of the tree already rules a match out: if x sits under a conjunction next to S, the value of x outside S cannot
// reach the root (the conjunction is false there whatever x says), and the same holds for the excluded side of a Filter outside its
// required side, through any number of operators above.  So the frequent leaves are decoded in a SECOND pass, and of their blocks only
// those whose docID range holds a set bit of a mask bitmap: the conjunction of the constraint subtrees on the leaf's path to the root,
// evaluated over the first-pass leaf bitmaps (any superset is a valid mask: an operand of a conjunction that is itself second-pass is
// left out, a disjunction with such an operand is not usable).  This is Conjuction::next's advance() on the longer list
// (docset_iterators.cpp:282-348) at block granularity.  The tree semantics used here are the compiler's (Compiler::node), from its
// effective root.  Layout of the program afterwards: [leaf markers] [mask operations, F_MASKOP] [the unchanged slot operations].
// Returns the number of slots the masks add.
static uint32_t flat_tree_masks(std::vector<DevStep> &steps, size_t begin, uint32_t nl, uint32_t slotsInUse, const trn_qnode *n, uint32_t nn, uint32_t root,
                                const std::vector<uint32_t> &leafNodes, const std::vector<DevTerm> &terms, uint32_t tileShift, double width) {
        if (leafNodes.size() != nl || nl > 16 || width <= 0)
                return 0;
        std::vector<int> leafOf(nn, -1), parent(nn, -1);
        for (uint32_t j = 0; j < nl; ++j)
                leafOf[leafNodes[j]] = int(j);
        {
                std::vector<uint32_t> st{root};
                while (!st.empty()) {
                        const uint32_t i = st.back();
                        st.pop_back();
                        if (n[i].kind == TRN_NODE_TERM)
                                continue;
                        for (uint32_t c = 0; c < n[i].nchildren; ++c) {
                                parent[n[i].first_child + c] = int(i);
                                st.push_back(n[i].first_child + c);
                        }
                }
        }
        auto blocksOf = [&](uint32_t j) -> double {
                const uint32_t t = n[leafNodes[j]].term;
                return t == kEmptyTerm ? 0.0 : double(terms[t].nblocks);
        };
        auto densOf = [&](uint32_t j) -> double {
                const uint32_t t = n[leafNodes[j]].term;
                return t == kEmptyTerm ? 0.0 : std::min(1.0, double(terms[t].documents) / width);
        };
        std::vector<uint8_t> masked(nl, 0);
        // density of the superset of node i computable from first-pass leaves (-1: unusable)
        std::function<double(uint32_t)> sup = [&](uint32_t i) -> double {
                const auto &X = n[i];
                switch (X.kind) {
                        case TRN_NODE_TERM:
                                return (leafOf[i] >= 0 && !masked[leafOf[i]]) ? densOf(uint32_t(leafOf[i])) : -1.0;
                        case TRN_NODE_AND: {
                                double d{1.0};
                                bool   any{false};
                                for (uint32_t c = 0; c < X.nchildren; ++c) {
                                        const double x = sup(X.first_child + c);
                                        if (x >= 0) {
                                                d *= x;
                                                any = true;
                                        }
                                }
                                return any ? d : -1.0;
                        }
                        case TRN_NODE_OR: {
                                double d{1.0};
                                for (uint32_t c = 0; c < X.nchildren; ++c) {
                                        const double x = sup(X.first_child + c);
                                        if (x < 0)
                                                return -1.0;
                                        d *= 1.0 - x;
                                }
                                return 1.0 - d;
                        }
                        case TRN_NODE_NOT:
                        case TRN_NODE_OPTIONAL:
                                return sup(X.first_child);
                        default:
                                return -1.0;
                }
        };
        // constraint subtrees of leaf j
        auto constraints = [&](uint32_t j) {
                std::vector<uint32_t> out;
                int                   c = int(leafNodes[j]);
                while (uint32_t(c) != root && parent[c] >= 0) {
                        const int   p = parent[c];
                        const auto &X = n[p];
                        if (X.kind == TRN_NODE_AND) {
                                for (uint32_t k = 0; k < X.nchildren; ++k)
                                        if (int(X.first_child + k) != c)
                                                out.push_back(X.first_child + k);
                        } else if (X.kind == TRN_NODE_NOT && int(X.first_child) + 1 == c)
                                out.push_back(X.first_child);
                        c = p;
                }
                return out;
        };
        const double W = double(1ull << tileShift);
        auto         need = [&](uint32_t j) { // estimated share of leaf j's blocks a mask leaves over
                double d{1.0};
                bool   any{false};
                for (auto cn : constraints(j)) {
                        const double x = sup(cn);
                        if (x >= 0) {
                                d *= x;
                                any = true;
                        }
                }
                if (!any)
                        return 1.0;
                const double span = width / std::max(1.0, blocksOf(j)); // docIDs a block covers
                return 1.0 - std::pow(1.0 - std::min(d, 1.0), span);
        };
        std::vector<uint32_t> order(nl);
        for (uint32_t j = 0; j < nl; ++j)
                order[j] = j;
        std::sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return blocksOf(a) > blocksOf(b); });
        bool anyMasked{false};
        for (auto j : order) {
                if (blocksOf(j) * W / width < 2.0)
                        break; // (sorted) blocks as wide as the tile: nothing to skip
                masked[j] = 1;
                if (need(j) > g_tree_mask_need)
                        masked[j] = 0;
                anyMasked |= masked[j] != 0;
        }
        for (auto j : order) // a later choice may have taken a constraint away
                if (masked[j] && need(j) > g_tree_mask_need + 0.15)
                        masked[j] = 0;
        if (!anyMasked)
                return 0;
        // ---- emission
        std::vector<DevStep>                      mops;
        std::unordered_map<uint32_t, int>         slotOfNode;
        std::map<std::vector<int>, int>           slotOfAnd;
        uint32_t                                  extra{0};
        const uint32_t                            kMaxExtra = 6;
        auto                                      newSlot   = [&]() -> int { return (extra < kMaxExtra && slotsInUse + extra < 30u) ? int(slotsInUse + extra++) : -1; };
        auto                                      op        = [&](uint8_t mode, int dst, int src) {
                DevStep S;
                std::memset(&S, 0, sizeof(S));
                S.op    = OP_SLOT;
                S.mode  = mode;
                S.dst   = uint8_t(dst);
                S.src   = uint8_t(src);
                S.flags = F_MASKOP;
                mops.push_back(S);
        };
        std::function<int(uint32_t)> emit = [&](uint32_t i) -> int { // slot holding a superset of node i, -1: unusable (or out of slots)
                const auto it = slotOfNode.find(i);
                if (it != slotOfNode.end())
                        return it->second;
                const auto &X = n[i];
                int         r{-1};
                if (X.kind == TRN_NODE_TERM)
                        r = (leafOf[i] >= 0 && !masked[leafOf[i]]) ? leafOf[i] : -1;
                else if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        r = emit(X.first_child);
                else if (X.kind == TRN_NODE_AND || X.kind == TRN_NODE_OR) {
                        std::vector<int> kids;
                        bool             ok{true};
                        for (uint32_t c = 0; c < X.nchildren && ok; ++c) {
                                const int k = sup(X.first_child + c) >= 0 ? emit(X.first_child + c) : -1;
                                if (k >= 0)
                                        kids.push_back(k);
                                else if (X.kind == TRN_NODE_OR)
                                        ok = false;
                        }
                        if (ok && kids.size() == 1)
                                r = kids[0];
                        else if (ok && kids.size() > 1) {
                                r = newSlot();
                                if (r >= 0) {
                                        op(M_SET, r, kids[0]);
                                        for (size_t k = 1; k < kids.size(); ++k)
                                                op(X.kind == TRN_NODE_AND ? M_AND : M_OR, r, kids[k]);
                                }
                        }
                }
                slotOfNode[i] = r;
                return r;
        };
        std::vector<int> maskSlot(nl, -1);
        for (uint32_t j = 0; j < nl; ++j) {
                if (!masked[j])
                        continue;
                std::vector<int> cs;
                for (auto cn : constraints(j))
                        if (sup(cn) >= 0) {
                                const int k = emit(cn);
                                if (k >= 0)
                                        cs.push_back(k);
                        }
                std::sort(cs.begin(), cs.end());
                cs.erase(std::unique(cs.begin(), cs.end()), cs.end());
                if (cs.empty()) {
                        masked[j] = 0; // (cannot be relied on by anybody: it was never usable)
                        continue;
                }
                int m;
                if (cs.size() == 1)
                        m = cs[0];
                else {
                        const auto it = slotOfAnd.find(cs);
                        if (it != slotOfAnd.end())
                                m = it->second;
                        else {
                                m = newSlot();
                                if (m >= 0) {
                                        op(M_SET, m, cs[0]);
                                        for (size_t k = 1; k < cs.size(); ++k)
                                                op(M_AND, m, cs[k]);
                                        slotOfAnd[cs] = m;
                                } else
                                        m = cs[0]; // out of slots: one constraint alone is a (weaker) mask
                        }
                }
                maskSlot[j] = m;
        }
        if (mops.size() > 32)
                return 0;
        anyMasked = false;
        for (uint32_t j = 0; j < nl; ++j)
                if (masked[j] && maskSlot[j] >= 0) {
                        steps[begin + j].flags |= F_MASKED;
                        steps[begin + j].src = uint8_t(maskSlot[j]);
                        anyMasked            = true;
                }
        if (!anyMasked)
                return 0;
        steps.insert(steps.begin() + std::ptrdiff_t(begin + nl), mops.begin(), mops.end());
        return extra;
}

extern "C" int trn_debug_compile(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, const trn_qnode *nodes, uint32_t nnodes,
                                 uint32_t root, int scored, trn_debug_step *out, uint32_t cap, uint32_t *nsteps, uint32_t *root_slot, uint32_t *nslots, char *err,
                                 size_t errcap) {
        static_assert(sizeof(trn_debug_step) == sizeof(DevStep), "trn_debug_step mirrors DevStep");
        auto seterr = [&](const std::string &m, int rc) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return rc;
        };
        if (!index || !terms || !nodes || !nnodes || !out || !nsteps || !root_slot || !nslots || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return seterr("bad arguments", TRN_ERR_ARG);
        BlockDirectory dir;
        try {
                std::vector<term_index_ctx> t(nterms);
                for (uint32_t i = 0; i < nterms; ++i) {
                        t[i].documents = terms[i].documents;
                        t[i].offset    = terms[i].chunk_off;
                        t[i].size      = terms[i].chunk_len;
                }
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, t.data(), nterms, 1, dir);
        } catch (const std::exception &e) {
                return seterr(e.what(), TRN_ERR_FORMAT);
        }
        std::vector<DevTerm> ht(nterms);
        for (uint32_t i = 0; i < nterms; ++i) {
                ht[i].documents = dir.terms[i].documents;
                ht[i].dir_begin = dir.terms[i].dir_begin;
                ht[i].nblocks   = dir.terms[i].nblocks;
                ht[i].first_doc = dir.terms[i].first_doc;
                ht[i].last_doc  = dir.terms[i].last_doc;
                ht[i].chunk_len = terms[i].chunk_len;
                ht[i].tf_begin  = dir.terms[i].tf_begin;
                ht[i].tf_base   = dir.terms[i].tf_base;
                ht[i].tf_shift  = dir.terms[i].tf_shift;
        }
        std::vector<DevStep> steps;
        Compiler             cc(nodes, nnodes, ht, scored == 1, root, steps);
        int                  rs = cc.run();
        if (rs < 0)
                return seterr(cc.err, cc.unsupported ? TRN_ERR_UNSUPPORTED : TRN_ERR_ARG);
        uint32_t treeLeaves{0};
        uint32_t maskSlots{0}, treeSlotsInUse{0};
        if (scored >= 2) { // DocumentsOnly program in its flat-tree form (what the second k_exec_docs launch runs); 3: with the masked second pass
                uint32_t root2 = uint32_t(rs);
                treeLeaves     = flat_tree_transform(steps, 0, cc.next_slot, ht, &cc.leaf_nodes, root2, treeSlotsInUse);
                if (treeLeaves)
                        rs = int(root2);
                if (scored == 3 && treeLeaves) {
                        uint32_t lo{0xffffffffu}, hi{0};
                        for (const auto &T : ht)
                                if (T.nblocks) {
                                        lo = std::min(lo, T.first_doc);
                                        hi = std::max(hi, T.last_doc);
                                }
                        if (hi >= lo)
                                maskSlots = flat_tree_masks(steps, 0, treeLeaves, treeSlotsInUse, nodes, nnodes, cc.root, cc.leaf_nodes, ht, 12, double(hi) - double(lo) + 1.0);
                }
        }
        if (steps.size() > cap)
                return seterr("step buffer too small", TRN_ERR_CAPACITY);
        std::memcpy(out, steps.data(), steps.size() * sizeof(DevStep));
        *nsteps    = uint32_t(steps.size());
        *root_slot = uint32_t(rs);
        *nslots    = (treeLeaves ? treeSlotsInUse + maskSlots : cc.next_slot) + 1; // + the scratch slot of the kernels
        return TRN_OK;
}

static void push_step(std::vector<DevStep> &steps, uint8_t op, uint8_t mode, uint32_t dst, uint32_t src, uint8_t flags, uint32_t term, double idf) {
        DevStep s;
        std::memset(&s, 0, sizeof(s));
        s.op    = op;
        s.mode  = mode;
        s.dst   = uint8_t(dst);
        s.src   = uint8_t(src);
        s.flags = flags;
        s.term  = term;
        s.idf   = idf;
        steps.push_back(s);
}

// =================================================================================================== exec
// small device scratch layout (d_small): [0] ticket u32, [2..3] seg_cursor u64, [4] overflow u32, then per-query arrays
static int exec_device_impl(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out, int set, cudaEvent_t k0, cudaEvent_t k1) {
        if (!c)
                return TRN_ERR_ARG;
        if (!c->have_index)
                return fail(c, TRN_ERR_STATE, "no index uploaded");
        if (!queries || !nq || mode < 0 || mode > 3)
                return fail(c, TRN_ERR_ARG, "trn_exec_batch: bad arguments");
        const bool compact = mode == TRN_MODE_DOCS_COMPACT; // DocumentsOnly with compact result segments; everything else is the same plan
        if (compact)
                mode = TRN_MODE_DOCS_ONLY;
        if (c->block_docs != (c->codec == TRN_CODEC_GOOGLE ? 32u : 128u))
                return fail(c, TRN_ERR_UNSUPPORTED, "the uploaded index was built with a block size other than the reference format's (decode sweep only)");
        if (mode == TRN_MODE_SCORED_TOPK && (k == 0 || k > kernel_max_k()))
                return fail(c, TRN_ERR_ARG, "top-k: k must be in [1, 512]");
        CK(cudaSetDevice(c->device));
        const bool scored = mode != TRN_MODE_DOCS_ONLY;
        // docID tile of this launch: set queries run one warp per tile (k_exec_docs) on larger tiles; scored queries keep a CTA-wide
        // fp32 score tile (k_exec_tiles).
        uint32_t execShift = scored ? c->tile_shift : c->docs_shift;
        execShift          = std::max(execShift, c->tile_shift);

        const double           tCompile0 = now_ms();
        std::vector<DevQuery>  hq(nq);
        std::vector<DevStep>   steps;
        std::vector<FlatQuery> fqs;    // queries k_score_flat runs
        std::vector<FlatLeaf>  leaves;
        uint64_t               genItems{0}, genItems2{0}, flatItems{0};
        uint32_t               treeSlots{1};
        uint32_t               maxRuns{0};
        uint32_t              maxSlots{1};
        bool                  anyCandidate{false}, anyMembership{false}, anyPhrase{false};
        uint64_t              items{0}, segCap{0}, candTotal{0}, postings{0}, bytes{0};
        for (uint32_t q = 0; q < nq; ++q) {
                const auto &Q = queries[q];
                if (!Q.nodes || !Q.nnodes)
                        return fail(c, TRN_ERR_ARG, "empty query");
                Compiler cc(Q.nodes, Q.nnodes, c->h_terms, scored, Q.root, steps);
                cc.allow_phrase = c->codec == TRN_CODEC_GOOGLE || c->have_hits; // GOOGLE: inline hits; LUCENE: hits.data uploaded (trn_upload_hits)
                auto &   dq     = hq[q];
                dq.step_begin   = uint32_t(steps.size());
                const int rs    = cc.run();
                anyPhrase |= cc.has_phrase;
                if (rs < 0)
                        return fail(c, cc.unsupported ? TRN_ERR_UNSUPPORTED : TRN_ERR_ARG, "query " + std::to_string(q) + ": " + cc.err);
                dq.nsteps    = uint32_t(steps.size()) - dq.step_begin;
                dq.root_slot = uint32_t(rs);
                dq.flat      = 0;
                {
                        // conjunction / disjunction whose operands are all terms (matchallterms / matchanyterms runs)
                        const auto &R = Q.nodes[cc.root];
                        if ((R.kind == TRN_NODE_AND || R.kind == TRN_NODE_OR) && R.nchildren <= 16) {
                                bool allTerms{true};
                                for (uint32_t ch = 0; ch < R.nchildren; ++ch)
                                        allTerms &= Q.nodes[R.first_child + ch].kind == TRN_NODE_TERM;
                                if (allTerms) {
                                        dq.flat = R.kind == TRN_NODE_AND ? 1u : 2u;
                                        if (R.kind == TRN_NODE_AND && R.nchildren <= 3)
                                                maxSlots = std::max<uint32_t>(maxSlots, R.nchildren); // one bitmap per operand
                                }
                        }
                }
                postings += cc.postings;
                bytes += cc.bytes;
                const Range r = cc.range(cc.root); // cc.root: the effective root (see apply_reference_root_filter_quirk)
                // Flat scored disjunction (a k-term OR / a single term, every leaf scoring with a weight >= +0.0) on the LUCENE codec:
                // k_score_flat (score_flat.cuh) instead of the step program
                bool flatScored{false};
                if (scored && c->flat_scored && c->codec == TRN_CODEC_LUCENE && execShift >= 13) {
                        const auto &R = Q.nodes[cc.root];
                        uint32_t    f0{cc.root}, nl{1};
                        bool        ok = R.kind == TRN_NODE_TERM;
                        if (R.kind == TRN_NODE_OR && R.nchildren <= score_flat_max_leaves()) {
                                ok = true;
                                f0 = R.first_child;
                                nl = R.nchildren;
                                for (uint32_t ch = 0; ch < nl; ++ch)
                                        ok &= Q.nodes[f0 + ch].kind == TRN_NODE_TERM;
                        }
                        for (uint32_t ch = 0; ok && ch < nl; ++ch) {
                                const double w = Q.nodes[f0 + ch].weight;
                                ok             = std::isfinite(w) && !std::signbit(w); // the -0.0f "untouched" sentinel of the score tile needs contributions >= +0.0
                        }
                        if (ok) {
                                flatScored = true;
                                steps.resize(dq.step_begin); // no step program
                                dq.nsteps = 0;
                                dq.flat   = 4u;
                                FlatQuery fq;
                                std::memset(&fq, 0, sizeof(fq));
                                fq.qid        = q;
                                fq.leaf_begin = uint32_t(leaves.size());
                                fq.nleaf      = nl;
                                for (uint32_t ch = 0; ch < nl; ++ch) {
                                        FlatLeaf L;
                                        L.term = Q.nodes[f0 + ch].term;
                                        L.pad  = 0;
                                        L.idf  = Q.nodes[f0 + ch].weight;
                                        leaves.push_back(L);
                                }
                                fqs.push_back(fq);
                        }
                }
                const uint32_t planSlots = cc.next_slot + 1; // + scratch slot (applied below, once the path of the query is known)
                // Candidate-driven evaluation (exec_docs_cand.cuh) when some term that EVERY match must hold is sparse: cost follows that
                // lead's postings (~cand_cost/2 warp-instructions per 32 candidates and probed term; the crossover was tuned on the and2
                // workload: 900 beats 450 and 1500) instead of the docID space (~1500 per tile + ~27 per block in it).
                // The boolean function of the tree over its (<= 8 distinct) terms is tabulated here; the device probes every term for
                // each candidate and looks the membership bits up.
                bool candidate{false};
                if (!scored && c->codec == TRN_CODEC_GOOGLE && c->cand_cost > 0 && !r.empty() && !cc.has_phrase) {
                        // distinct non-empty terms below the effective root (at most 8)
                        uint32_t tv[8];
                        uint32_t n{0};
                        bool     small{true};
                        {
                                uint32_t stack[64], sp{0};
                                stack[sp++] = cc.root;
                                while (sp && small) {
                                        const auto &X = Q.nodes[stack[--sp]];
                                        if (X.kind == TRN_NODE_TERM) {
                                                if (X.term == kEmptyTerm || !c->h_terms[X.term].nblocks)
                                                        continue;
                                                bool seen{false};
                                                for (uint32_t j = 0; j < n; ++j)
                                                        seen |= tv[j] == X.term;
                                                if (!seen) {
                                                        if (n == 8)
                                                                small = false;
                                                        else
                                                                tv[n++] = X.term;
                                                }
                                        } else if (sp + X.nchildren > 64)
                                                small = false;
                                        else
                                                for (uint32_t k = 0; k < X.nchildren; ++k)
                                                        stack[sp++] = X.first_child + k;
                                }
                        }
                        small = small && n >= 2;
                        if (small) {
                                // truth vectors: bit `bits` of vec(node) = value of the node under the term assignment `bits` (bit j = tv[j])
                                uint8_t  truth[256];
                                uint32_t necessary{(1u << n) - 1u};
                                bool     any{false};
                                if (dq.flat == 1u && n == Q.nodes[cc.root].nchildren) { // all-term conjunction: only the all-ones assignment matches
                                        std::memset(truth, 0, sizeof(truth));
                                        truth[(1u << n) - 1u] = 1;
                                        any                   = true;
                                } else {
                                        const TruthVec tvec = truth_vector(Q.nodes, cc.root, tv, n);
                                        for (uint32_t bits = 0; bits < (1u << n); ++bits) {
                                                truth[bits] = uint8_t((tvec.w[bits >> 6] >> (bits & 63u)) & 1ull);
                                                if (truth[bits]) {
                                                        necessary &= bits;
                                                        any = true;
                                                }
                                        }
                                }
                                if (any && necessary) {
                                        // probe order: the lead (rarest necessary term), the other necessary terms rarest first (they filter),
                                        // then the rest
                                        uint32_t order[8], nn{0}, no{0};
                                        for (uint32_t j = 0; j < n; ++j)
                                                if ((necessary >> j) & 1u)
                                                        order[no++] = j;
                                        nn = no;
                                        for (uint32_t j = 0; j < n; ++j)
                                                if (!((necessary >> j) & 1u))
                                                        order[no++] = j;
                                        auto byBlocks = [&](uint32_t x, uint32_t y) { return c->h_terms[tv[x]].nblocks < c->h_terms[tv[y]].nblocks; };
                                        std::sort(order, order + nn, byBlocks);
                                        std::sort(order + nn, order + n, byBlocks);
                                        const uint32_t lead = tv[order[0]];
                                        double         blocks{0};
                                        for (uint32_t j = 0; j < n; ++j)
                                                blocks += c->h_terms[tv[j]].nblocks;
                                        const double width   = double(c->max_docid) - double(std::min(c->min_docid, c->max_docid)) + 1.0; // docID span of THIS source
                                        const double perTile = double(1ull << execShift) / width;
                                        const double lhs     = double(n - 1) * c->h_terms[lead].nblocks * perTile * double(c->cand_cost);
                                        const double rhs     = 1500.0 + (dq.flat == 1u ? 0.0 : 150.0 * n) + blocks * perTile * (dq.flat == 1u ? 27.0 : 35.0);
                                        if (lhs < rhs) {
                                                // replace the step program: terms in probe order, then the truth table re-indexed to probe positions
                                                steps.resize(dq.step_begin);
                                                for (uint32_t j = 0; j < n; ++j)
                                                        push_step(steps, OP_LEAF, M_NONE, 0, 0, 0, tv[order[j]], 0.0);
                                                uint32_t words[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                                                for (uint32_t pb = 0; pb < (1u << n); ++pb) { // pb: bit j = term at probe position j
                                                        uint32_t bits{0};
                                                        for (uint32_t j = 0; j < n; ++j)
                                                                if ((pb >> j) & 1u)
                                                                        bits |= 1u << order[j];
                                                        if (truth[bits])
                                                                words[pb >> 5] |= 1u << (pb & 31u);
                                                }
                                                for (uint32_t w = 0; w < 8; w += 4) {
                                                        DevStep st;
                                                        std::memset(&st, 0, sizeof(st));
                                                        st.op   = OP_TABLE;
                                                        st.dst  = uint8_t(w);
                                                        st.term = words[w];
                                                        st.pad2 = words[w + 1];
                                                        uint64_t hi = uint64_t(words[w + 2]) | (uint64_t(words[w + 3]) << 32);
                                                        std::memcpy(&st.idf, &hi, 8);
                                                        steps.push_back(st);
                                                }
                                                dq.nsteps    = uint32_t(steps.size()) - dq.step_begin;
                                                dq.root_slot = nn;
                                                candidate    = true;
                                                dq.flat      = 3u;
                                                dq.tile_lo   = 0;
                                                dq.ntiles    = (c->h_terms[lead].nblocks + 31u) / 32u;
                                                anyCandidate = true;
                                                anyMembership |= nn < n;
                                        }
                                }
                        }
                }
                // Flat-tree path (exec_docs_flat.cuh): a DocumentsOnly tree that is neither an all-term run nor candidate-driven decodes ALL its
                // leaves of a tile in one flat (leaf, block) pass — each leaf into a bitmap of its own — and then runs slot operations only.
                // The per-leaf groups of the step-program path ran at a third of the lanes with up to 8 live bitmaps per warp; here
                // the lanes are packed across leaves, and a smaller tile pays for the extra bitmaps.
                bool treeFlat{false};
                if (!scored && !candidate && dq.flat == 0u && c->codec == TRN_CODEC_GOOGLE && c->tree_shift && !r.empty() && !cc.has_phrase) {
                        uint32_t       root2 = dq.root_slot, inUse{0};
                        const uint32_t nl    = flat_tree_transform(steps, dq.step_begin, cc.next_slot, c->h_terms, &cc.leaf_nodes, root2, inUse);
                        if (nl) {
                                uint32_t extra{0};
                                if (c->tree_masks) {
                                        const double width = double(c->max_docid) - double(std::min(c->min_docid, c->max_docid)) + 1.0; // docID span of THIS source
                                        extra = flat_tree_masks(steps, dq.step_begin, nl, inUse, Q.nodes, Q.nnodes, cc.root, cc.leaf_nodes, c->h_terms, c->tree_shift, width);
                                }
                                dq.nsteps = uint32_t(steps.size()) - dq.step_begin;
                                dq.root_slot = root2;
                                dq.flat      = 5u;
                                treeSlots    = std::max(treeSlots, inUse + extra);
                                treeFlat  = true;
                        }
                }
                if (!flatScored && !treeFlat)
                        maxSlots = std::max(maxSlots, planSlots);
                if (candidate) {
                } else if (r.empty()) {
                        dq.tile_lo = 0;
                        dq.ntiles  = 0;
                } else {
                        const uint32_t qshift = flatScored ? c->scored_shift : (treeFlat ? c->tree_shift : execShift); // per-path tile
                        dq.tile_lo            = r.lo >> qshift;
                        dq.ntiles             = (r.hi >> qshift) - dq.tile_lo + 1;
                }
                dq.item_base = uint32_t(items);
                dq.gen_base  = uint32_t(genItems);
                dq.gen_base2 = uint32_t(genItems2);
                items += dq.ntiles;
                if (treeFlat)
                        genItems2 += dq.ntiles;
                else if (!flatScored)
                        genItems += dq.ntiles;
                if (items >= (1ull << 32))
                        return fail(c, TRN_ERR_CAPACITY, "batch has more than 2^32 (query, tile) work items; split it");
                const uint64_t width = r.empty() ? 0 : uint64_t(r.hi) - r.lo + 1;
                segCap += std::min(cc.bound(cc.root), width);
                dq.cand_base = uint32_t(candTotal);
                dq.cand_cap  = uint32_t(std::min<uint64_t>(uint64_t(dq.ntiles) * k, 0xffffffffull));
                if (flatScored) {
                        auto &fq      = fqs.back();
                        fq.tile_lo    = dq.tile_lo;
                        fq.ntiles     = dq.ntiles;
                        fq.nruns      = (dq.ntiles + c->run_tiles - 1u) / c->run_tiles;
                        fq.item_base  = dq.item_base;
                        fq.local_base = uint32_t(flatItems);
                        flatItems += dq.ntiles;
                        maxRuns     = std::max(maxRuns, fq.nruns);
                        dq.cand_cap = uint32_t(std::min<uint64_t>(uint64_t(fq.nruns) * k, 0xffffffffull));
                        fq.cand_base = dq.cand_base;
                        fq.cand_cap  = dq.cand_cap;
                }
                if (mode == TRN_MODE_SCORED_TOPK) {
                        candTotal += dq.cand_cap;
                        if (candTotal >= (1ull << 32))
                                return fail(c, TRN_ERR_CAPACITY, "top-k candidate space exceeds 2^32 entries; split the batch");
                }
        }
        c->tm.host_compile_ms += float(now_ms() - tCompile0);
        const double   tEnqueue0  = now_ms();
        const uint32_t totalItems = uint32_t(items);
        if (anyCandidate) { // the candidate array + one gather buffer must fit a warp's share of shared memory
                const uint32_t slotBytes = (1u << execShift) / 8u, stageB = exec_docs_stage_bytes(), need = exec_docs_cand_smem_bytes(anyMembership);
                if (need > stageB)
                        maxSlots = std::max(maxSlots, (need - stageB + slotBytes - 1u) / slotBytes);
        }

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
                CK(c->d_cand.ensure(std::max<size_t>(8, candTotal * 8)));
                CK(c->d_topk_docids.ensure(size_t(nq) * k * 4));
                CK(c->d_topk_scores.ensure(size_t(nq) * k * 4));
                CK(c->d_topk_counts.ensure(size_t(nq) * 4));
        }
        const uint32_t nflat = uint32_t(fqs.size());
        if (nflat) {
                CK(c->d_fq.ensure(fqs.size() * sizeof(FlatQuery)));
                CK(c->d_leaves.ensure(leaves.size() * sizeof(FlatLeaf)));
                CK(c->d_luts.ensure(leaves.size() * 64 * sizeof(float)));
                CK(cudaMemcpyAsync(c->d_fq.p, fqs.data(), fqs.size() * sizeof(FlatQuery), cudaMemcpyHostToDevice, c->stream));
                CK(cudaMemcpyAsync(c->d_leaves.p, leaves.data(), leaves.size() * sizeof(FlatLeaf), cudaMemcpyHostToDevice, c->stream));
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
                        const DevQuery &dq = hq[q];
                        qi[q] = trn_qitems{dq.item_base, dq.ntiles, dq.tile_lo, dq.flat == 5u ? c->tree_shift : execShift};
                }
        }
        CK(cudaMemcpyAsync(c->d_queries.p, hq.data(), nq * sizeof(DevQuery), cudaMemcpyHostToDevice, c->stream));
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
        P.gen_items    = uint32_t(genItems);
        P.has_phrase   = anyPhrase ? 1u : 0u;
        P.nslots       = maxSlots;
        P.exec_shift   = execShift;
        P.stage_bytes  = exec_stage_bytes(c->codec);
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
                const uint64_t ownItems   = genItems; // tickets of the step-program launch
                CK(cudaEventRecord(k0, c->stream));
                if (nflat && flatItems) {
                        // flat scored disjunctions: per-leaf BM25 tables once per batch, then k_score_flat
                        ScoreParams S;
                        std::memset(&S, 0, sizeof(S));
                        S.ix           = P.ix;
                        S.fq           = c->d_fq.as<FlatQuery>();
                        S.leaves       = c->d_leaves.as<FlatLeaf>();
                        S.luts         = c->d_luts.as<float>();
                        S.nflat        = nflat;
                        S.run_tiles    = c->run_tiles;
                        S.total_items  = mode == TRN_MODE_SCORED_TOPK ? uint32_t(std::min<uint64_t>(uint64_t(maxRuns) * nflat, 0xffffffffull)) : uint32_t(flatItems);
                        S.tile_shift   = c->scored_shift;
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
                        if (uint64_t(maxRuns) * nflat >= (1ull << 32))
                                return fail(c, TRN_ERR_CAPACITY, "batch has more than 2^32 (run, query) work items; split it");
                        CK(launch_build_luts(S.leaves, uint32_t(leaves.size()), c->d_luts.as<float>(), c->stream));
                        CK(launch_score_flat(S, c->flat_threads, c->num_sms, c->stream));
                        launches += 2;
                }
                if (ownItems) {
                        const int perSM = warpKernel ? exec_docs_max_ctas_per_sm(execShift, maxSlots, exec_docs_stage_bytes(), false, c->codec == TRN_CODEC_LUCENE) : exec_max_ctas_per_sm(execShift, maxSlots, mode, c->codec);
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
                if (warpKernel && genItems2) { // flat-tree plans: same kernel, own tile size / slot count / ticket space
                        ExecParams P2 = P;
                        P2.exec_shift = c->tree_shift;
                        P2.nslots     = treeSlots;
                        P2.gen_items  = uint32_t(genItems2);
                        P2.gen_sel    = 1;
                        P2.ticket     = reinterpret_cast<uint32_t *>(small + 4);
                        const int perSM = exec_docs_max_ctas_per_sm(P2.exec_shift, P2.nslots, exec_docs_stage_bytes(), true);
                        if (perSM <= 0)
                                return fail(c, TRN_ERR_CUDA, "the flat-tree launch does not fit on an SM with this many docset slots");
                        const int grid = int(std::min<uint64_t>(uint64_t(c->num_sms) * perSM, std::max<uint64_t>(1, (genItems2 + 3) / 4)));
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
        c->last_postings = postings;
        c->last_bytes    = bytes;
        if (out) {
                std::memset(out, 0, sizeof(*out));
                out->nq                  = nq;
                out->postings_scanned    = postings;
                out->index_bytes_touched = bytes;
                out->kernel_launches     = launches;
        }
        return TRN_OK;
}

extern "C" int trn_exec_batch_device(trn_ctx *c, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out) {
        if (!c)
                return TRN_ERR_ARG;
        CK(cudaSetDevice(c->device));
        c->have_kernel_events = false;
        c->tm                 = trn_timings{};
        const double t0       = now_ms();
        CK(cudaEventRecord(c->ev0, c->stream));
        const int r = exec_device_impl(c, queries, nq, mode, k, out, 0, c->evk0, c->evk1);
        c->tm.total_ms = float(now_ms() - t0);
        if (r != TRN_OK)
                return r;
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
                const int  r = exec_device_impl(c, queries + ch[i].q0, ch[i].n, mode, k, &part, set, c->ev_ck0[i % 16], c->ev_ck1[i % 16]);
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
        c->last_mode = -1;
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
        const bool               legacyDecode = (decodeKernel == "legacy" || decodeKernel == "single-pass") && c->block_docs == (c->codec == TRN_CODEC_GOOGLE ? 32u : 128u);
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
                units += (legacyDecode && c->codec == TRN_CODEC_LUCENE) ? t.nblocks : (t.nblocks + 31) / 32;
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
                                D.last_n      = (g0 + D.cnt == t.nblocks && (c->codec == TRN_CODEC_GOOGLE ? true : lastN != bd)) ? lastN : 0u;
                                if (c->codec == TRN_CODEC_LUCENE && (t.documents & 127u) == 0u)
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
                else if (c->codec == TRN_CODEC_GOOGLE && (materialise || forceNew))
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
