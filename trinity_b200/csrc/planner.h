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
        uint32_t tile_shift{13};   // TRN_TILE_SHIFT: directory granularity == scored tile (8192 docs, the reference's window docset_spans.h:74)
        uint32_t docs_shift{14};   // TRN_DOCS_SHIFT: docID tile (log2) of the warp-per-tile DocumentsOnly kernel
        uint32_t tree_shift{13};   // TRN_TREE_SHIFT: docID tile (log2) of the flat-tree launch of k_exec_docs (0 = flat-tree path off)
        uint32_t scored_shift{13}; // TRN_SCORED_SHIFT: log2 of k_score_flat's tile (13 = the reference's window, 14)
        uint32_t run_tiles{128};   // TRN_RUN_TILES: consecutive tiles per work item of the flat scored kernel (top-k state lives across a run)
        int      cand_cost{900};   // TRN_CAND_COST: modelled warp-instructions per 32 candidates of the candidate-driven conjunction (0 = never use it)
        bool     flat_scored{true}; // TRN_FLAT_SCORED=0: every scored query through the general step-program kernel (A/B switch)
        bool     tree_masks{false}; // TRN_TREE_MASKS=1: flat-tree queries decode their frequent leaves in a masked second pass (flat_tree_masks). It
                                    // halves the DRAM bytes, but the needed blocks of a tile fill a fraction of a 32-lane group, so the warp-instruction
                                    // count does not drop and the benchmark's trees ran slower with it. Off by default. (Not a matter of WHICH leaves
                                    // are admitted — TRN_TREE_MASK_NEED does not recover it: a few masked queries raise the launch-wide slot count and
                                    // take resident warps from every query.)
        double   tree_mask_need{0.6}; // TRN_TREE_MASK_NEED: a leaf is decoded in the masked pass when at most this share of its blocks is expected to survive its mask
        bool     allow_phrase{false}; // the kernels execute OP_PHRASE (GOOGLE: inline hits; LUCENE: once hits.data is uploaded)
        // kernel limits (kernels.h)
        uint32_t score_flat_max_leaves{0};          // leaves of a k_score_flat query
        uint32_t docs_stage_bytes{0};               // per-warp staging bytes of k_exec_docs
        uint32_t cand_smem_bytes[2]{0, 0};          // per-warp shared memory of the candidate-driven path, [with membership bits]
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
        uint64_t               seg_cap{0};     // upper bound of the batch's matches (result segments)
        uint64_t               cand_total{0};  // top-k candidate entries
        uint64_t               postings{0}, bytes{0};
        bool                   any_phrase{false};
};

// Plans a batch (mode: TRN_MODE_*; k: top-k).  Returns TRN_OK, or an error code with its message in err: TRN_ERR_ARG /
// TRN_ERR_UNSUPPORTED for a plan the compiler refuses, TRN_ERR_CAPACITY when the batch has to be split.
int plan_batch(const PlanConfig &cfg, const std::vector<DevTerm> &terms, const trn_query *queries, uint32_t nq, int mode, uint32_t k, BatchPlan &out,
               std::string &err);

// the block directory of an index (throws what build_block_directory throws)
void build_directory(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, int threads, BlockDirectory &dir);
// the device term table of a directory
std::vector<DevTerm> dev_terms(const BlockDirectory &dir, const trn_term *terms, uint32_t nterms);
// min_docid: the smallest docID a term holds (0xffffffff: none); max_docid == 0 (not recorded, e.g. a segment directory): the largest
void docid_span(const std::vector<DevTerm> &terms, uint32_t &min_docid, uint32_t &max_docid);

} // namespace trn
