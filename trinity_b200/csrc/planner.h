// Host-side batch planner: compiles every plan of a batch into its step program and decides the path (TRN_ROUTE_*) each query runs,
// with the tile ranges, ticket spaces and buffer bounds of the launches.  A pure function of the plans, the index's term table and a
// PlanConfig — no CUDA call — so the engine calls it before it sizes buffers and launches, and the decision is pinned on the CPU
// (trn_debug_plan, tests/test_plan_routes_cpu.py).  Host only.
#pragma once
#include "../../include/trinity_b200.h"
#include "codecs.h"
#include "device_types.h"
#include <string>
#include <vector>

namespace trn {

struct PlanConfig {
        // the uploaded index (trn_upload_index)
        int      codec{0};
        uint32_t min_docid{1}; // smallest docID any term holds (a docID-range shard does not start at 1)
        uint32_t max_docid{0};
        // knobs (plan_config_from_env)
        uint32_t tile_shift{13};   // directory granularity == scored tile (8192 docs, the reference's window docset_spans.h:74); not read from the environment
        uint32_t docs_shift{14};   // TRN_DOCS_SHIFT: docID tile (log2) of the warp-per-tile DocumentsOnly kernel
        uint32_t tree_shift{13};   // TRN_TREE_SHIFT: docID tile (log2) of the flat-tree launch of k_exec_docs (0 = flat-tree path off)
        uint32_t scored_shift{13}; // TRN_SCORED_SHIFT: log2 of k_score_flat's tile (13 = the reference's window, 14)
        uint32_t run_tiles{128};   // TRN_RUN_TILES: consecutive tiles per work item of the flat scored kernel (top-k state lives across a run)
        int      cand_cost{900};   // TRN_CAND_COST: modelled warp-instructions per 32 candidates of the candidate-driven conjunction (0 = never use it)
        bool     flat_scored{true}; // TRN_FLAT_SCORED=0: every scored query through the general step-program kernel (A/B switch)
        bool     allow_phrase{false}; // the kernels execute OP_PHRASE (GOOGLE: inline hits; LUCENE: once hits.data is uploaded)
        bool     dense_bitmaps{true}; // TRN_DENSE_BITMAPS=0: no resident docID bitmaps of dense terms (select_dense_terms)
        double   dense_budget{0.25};  // TRN_DENSE_BUDGET: the bitmaps of one source take at most this share of its index bytes (0 .. 1)
        bool     probe_bitmaps{true}; // TRN_PROBE_BITMAPS=0: no probe bitmaps (select_probe_terms); TRN_DENSE_BITMAPS=0 turns them off too
        double   probe_ratio{16.0};   // TRN_PROBE_RATIO: a probe bitmap is at most this many times its term's chunk
        double   probe_budget{2.0};   // TRN_PROBE_BUDGET: the probe bitmaps of one source take at most this multiple of its index bytes (0: none)
        bool     dense_runs{true};    // TRN_DENSE_RUNS=0: all-bitmap flat ANDs take (query, tile) tickets like the other flat ANDs (BatchPlan::dense_runs)
        bool     mixed_runs{true};    // TRN_MIXED_RUNS=0: flat ANDs with one decoded operand take (query, tile) tickets (BatchPlan::mixed_runs)
        bool     cand_runs{true};     // TRN_CAND_RUNS=0: candidate-driven groups take tickets in query order (BatchPlan::cand_runs)
        // kernel limits (kernels.h)
        uint32_t score_flat_max_leaves{0};          // leaves of a k_score_flat query
        uint32_t docs_stage_bytes{0};               // per-warp staging bytes of k_exec_docs
        uint32_t cand_smem_bytes[2]{0, 0};          // per-warp shared memory of the candidate-driven path, [with membership bits]
        uint32_t mixed_smem_bytes{0};               // per-warp shared memory of the mixed flat ANDs' run tickets
};

// the knobs of PlanConfig from the environment (the index fields and the kernel limits keep their defaults)
PlanConfig plan_config_from_env();

struct BatchPlan {
        std::vector<DevQuery>  queries; // DevQuery::route: the path of every query
        std::vector<DevStep>   steps;
        std::vector<FlatQuery> flat; // queries k_score_flat runs
        std::vector<FlatLeaf>  leaves;
        uint32_t               exec_shift{0};  // docID tile (log2) of the step-program launch (k_exec_docs / k_exec_tiles)
        uint32_t               nslots{1};      // docset slots of the step-program launch
        uint32_t               tree_slots{1};  // docset slots of the flat-tree launch of k_exec_docs
        uint32_t               max_runs{0};    // most runs of one k_score_flat query
        uint64_t               items{0};       // (query, tile) work items of the batch
        uint64_t               gen_items{0}, gen_items2{0}, flat_items{0}; // tickets of the step-program, flat-tree and k_score_flat launches
        // flat ANDs whose operands all have a resident bitmap (DocumentsOnly, no phrase plan in the batch): one ticket per (query, 2^17-docID
        // run) pair, {query, first tile} (dense_run_end: device_types.h), ordered run-major, in front of the step-program launch's gen_items
        std::vector<uint2>     dense_runs;
        // flat ANDs with exactly one operand without a resident bitmap (the lead, decoded; the others probed in their bitmaps), same
        // conditions: the same {query, first tile} tickets over the same runs, run-major, between dense_runs and gen_items
        std::vector<uint2>     mixed_runs;
        // candidate-driven queries, same conditions: one ticket {query, group} per 32-block group of the lead, counting-sorted by the
        // 2^kDenseAlignShift-docID run of the group's first docID (ties in query order), between mixed_runs and gen_items.  The queries
        // that run in flight together then probe the same runs of the resident bitmaps.  A group keeps its item, item_base + group.
        std::vector<uint2>     cand_runs;
        // what the launch reads of them: per ticket the group's own step-program ticket, gen_base + group (the launch skips those
        // tickets where the step-program tickets reach the candidate-driven queries)
        std::vector<uint32_t>  cand_order;
        uint64_t               seg_cap{0};     // upper bound of the batch's matches (result segments)
        uint64_t               cand_total{0};  // top-k candidate entries
        uint64_t               postings{0}, bytes{0};
        bool                   any_phrase{false};
        struct CollectPlan {   // TRN_MODE_MATCHED_TERMS: what the collect pass runs per match (plan_collect)
                std::vector<CollectQuery>  queries;
                std::vector<uint32_t>      terms;
                std::vector<CollectPhrase> phrases;
                std::vector<DevStep>       args;
                std::vector<CollectOp>     prog;
        } collect;
};
using CollectPlan = BatchPlan::CollectPlan;

// The structural checks every plan passes before it is compiled: root in range, depth <= 64, children behind their parent, a tree, term
// ids below nterms (or kEmptyTerm), phrases of 2..16 terms.  A phrase when !allow_phrase sets `unsupported`; has_phrase reports one.
bool validate_plan(const trn_qnode *nodes, uint32_t nn, uint32_t root, uint32_t nterms, bool allow_phrase, std::string &err, bool &unsupported, bool &has_phrase);

// The collect programs of a batch in the default exec mode (TRN_MODE_MATCHED_TERMS): per query its distinct terms (at most 32, ascending
// term index), its phrase nodes (at most 32) and its nodes in post order.  TRN_ERR_UNSUPPORTED beyond those limits.
int plan_collect(const std::vector<DevTerm> &terms, const trn_query *queries, uint32_t nq, CollectPlan &out, std::string &err);

// Plans a batch (mode: TRN_MODE_*; k: top-k; TRN_MODE_MATCHED_TERMS: the DocumentsOnly program without the root-filter quirk, plus
// BatchPlan::collect).  dense_off: per term, the first word of its resident bitmap (DenseSelection::off), or
// null when the source has none.  Returns TRN_OK, or an error code with its message in err: TRN_ERR_ARG / TRN_ERR_UNSUPPORTED for a
// plan the compiler refuses, TRN_ERR_CAPACITY when the batch has to be split.  clip (null: none): per query the inclusive docID span its
// matches can lie in (its allow set's first and last docID; x > y: none), to which its tile range is clipped.  groups (null: candidate-driven
// queries keep query-order tickets): the first docID of every lead group (group_starts), which orders BatchPlan::cand_runs.
//
// GroupStarts: the first docID of every 32-block group of every term (GOOGLE directories), where a candidate-driven work item starts.
// Group g of term t is first[base[t] + g]: the last docID of block 32g - 1 plus one, the term's first docID for g = 0.  1/32 of the
// directory's entries.
struct GroupStarts {
        std::vector<uint32_t> base; // per term: its first entry in `first`
        std::vector<uint32_t> first;
};
GroupStarts group_starts(const BlockDirectory &dir);
int plan_batch(const PlanConfig &cfg, const std::vector<DevTerm> &terms, const uint32_t *dense_off, const trn_query *queries, uint32_t nq, int mode,
               uint32_t k, BatchPlan &out, std::string &err, const uint2 *clip = nullptr, const GroupStarts *groups = nullptr);

// Resident docID bitmaps of dense terms (GOOGLE sources; LUCENE sources get none).  A selected term owns one bitmap over its own docID
// span, both ends aligned to 2^kDenseAlignShift docIDs — the largest tile of any k_exec_docs launch — so every tile of every launch lies
// wholly inside the bitmap or holds none of the term's documents (kDenseAlignShift, kDenseNone: device_types.h).
struct DenseSelection {
        std::vector<uint32_t> off;  // per term: its first word in the bitmap array, kDenseNone when it has no bitmap
        std::vector<uint32_t> order; // the selected terms, densest first (the order their bitmaps are laid out in)
        uint64_t              words{0};
};
// first docID and 32-bit words of term T's bitmap (64-bit arithmetic: the span of a term ending at 2^32 - 2 ends at 2^32)
void dense_span(const DevTerm &T, uint64_t &base, uint64_t &words);
// A term qualifies when its bitmap is no larger than its chunk (chunk_len); qualifying terms are taken densest first (ties: lower term
// id) while their bitmaps fit into cfg.dense_budget x index_bytes.  Reads the term records and the config only.
DenseSelection select_dense_terms(const PlanConfig &cfg, const std::vector<DevTerm> &terms, uint64_t index_bytes);

// The second tier, the probe bitmaps, which only the candidate-driven conjunction reads: a probe there tests one word, so a bitmap pays
// off far below the density at which the flat paths, which read whole bitmaps, gain from one.  A GOOGLE term without a dense bitmap
// qualifies when its bitmap is at most cfg.probe_ratio x its chunk; qualifying terms are taken densest first (ties: lower term id) while
// the tier fits into cfg.probe_budget x index_bytes and both tiers together into fewer than 2^32 words (the offsets are 32-bit word
// indices).  The tier is laid out behind the dense bitmaps.  off: per term, its dense.off entry when it has a dense bitmap, its first
// word in the bitmap array when it has a probe bitmap, kDenseNone otherwise; order and words: the probe tier alone.
DenseSelection select_probe_terms(const PlanConfig &cfg, const std::vector<DevTerm> &terms, uint64_t index_bytes, const DenseSelection &dense);

// the block directory of an index (throws what build_block_directory throws)
void build_directory(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, int threads, BlockDirectory &dir);
// the device term table of a directory
std::vector<DevTerm> dev_terms(const BlockDirectory &dir, const trn_term *terms, uint32_t nterms);
// min_docid: the smallest docID a term holds (0xffffffff: none); max_docid == 0 (not recorded, e.g. a segment directory): the largest
void docid_span(const std::vector<DevTerm> &terms, uint32_t &min_docid, uint32_t &max_docid);

} // namespace trn
