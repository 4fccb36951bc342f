// Device-side data layout shared by the host (planner.cpp, engine.cu) and kernels.cu (device).
#pragma once
#include "../../include/trinity_b200.h"
#include <cstdint>
#include <vector_types.h>

namespace trn {

struct HitTerm;

static constexpr uint32_t kEmptyTerm = 0xffffffffu;

// one per dictionary term (36 B)
struct DevTerm {
        uint32_t documents;
        uint32_t dir_begin; // first entry in blk_last / blk_off (nblocks + 1 entries incl. sentinel)
        uint32_t nblocks;
        uint32_t first_doc;
        uint32_t last_doc;
        uint32_t chunk_len;
        // sparse docID -> block table (codecs.h): tile_first[tf_begin + j] = first block whose last docID >= (tf_base + j) << tf_shift,
        // j = 0 .. (last_doc >> tf_shift) - tf_base + 1; tf_shift == 32: the term has no table (few blocks: search blk_last directly)
        uint32_t tf_begin;
        uint32_t tf_base;
        uint32_t tf_shift;
};
static_assert(sizeof(DevTerm) == 36, "DevTerm layout (BlockDirectory::bytes counts 36 B per term)");

struct DevIndex {
        const uint8_t * index;    // raw reference-format bytes (google index / lucene index), 256B aligned, 64B tail padding
        const uint32_t *blk_last; // last docID per block (+ sentinel UINT32_MAX per term)
        const uint32_t *blk_off;  // payload byte offset per block (+ sentinel = end of block area)
        const DevTerm * terms;
        const uint32_t *masked;     // optional docID bitmap of masked (deleted/updated) documents, word i = docIDs [32i, 32i+32)
        const uint32_t *tile_first; // per-term sparse docID -> block tables (DevTerm::tf_*)
        uint32_t        nterms;
        uint32_t        ntiles;     // number of 2^tile_shift-document tiles of the docID space
        uint32_t        tile_shift; // tile of the scored kernel (8192 documents: the reference's window, docset_spans.h:74)
        uint32_t        max_docid;
        uint32_t        block_docs; // documents per full block (GOOGLE: google_codec.h:18 N = 32 — other values only for the decode sweep; LUCENE: 128)
        int             codec;
        // LUCENE positions (trn_upload_hits; null otherwise): hits.data and its load-time directory (codecs.h HitsDirectory)
        const uint8_t * hits;
        const uint32_t *hit_base; // parallel to blk_last: hits of the term's documents before the block
        const uint32_t *hblk_off; // per term: byte offsets of its 128-hit blocks in hits.data, then of its varbyte tail, then the end
        const struct HitTerm *hit_term; // per term: {first entry in hblk_off, sumHits} (hitcursor.h)
};

// ---- per-query step program (built on the host from the trn_qnode tree) ----
enum StepOp : uint8_t {
        OP_LEAF      = 0, // decode term, combine its docset into slot dst (mode), optionally accumulate BM25 (flag SCORE)
        OP_SLOT      = 1, // combine slot src into slot dst (mode)
        OP_CLEAR     = 2, // dst = 0
        OP_LEAFSCORE = 3, // second pass: decode term, accumulate BM25 where slot src (mask) has the doc's bit
        OP_COUNT_ADD = 4, // bit-sliced saturating counter in slots dst .. dst+mode-1 (LSB first) += slot src   (DisjunctionSome)
        OP_COUNT_GE  = 5, // dst = documents whose counter (slots src .. src+mode-1) is >= term (min-should-match)
        OP_PHRASE    = 7, // phrase.cuh: keep the documents of slot dst that hold the phrase whose `mode` term ids follow in OP_ARG steps (four per
                          // step); flag F_SCORE: add score(matchCnt, idf) (idf = the sum of the terms' weights) to the score tile
        OP_ARG       = 8, // operand words of the preceding step (never executed)
        OP_TABLE     = 6, // candidate-driven trees: 4 words of the query's truth table (term, pad2, idf as two words); dst = first word index
};
enum StepMode : uint8_t { M_SET = 0, M_OR = 1, M_AND = 2, M_ANDNOT = 3, M_NONE = 4 };
// encodings of a compact result segment (trn_result::item_desc bits 30-31 == TRN_ENC_*)
static constexpr uint32_t kEncU32 = 0, kEncU16 = 1, kEncBitmap = 2, kEncU8B = 3;

enum StepFlags : uint8_t {
        F_SCORE          = 1,
        F_BREAK_IF_EMPTY = 2,
        F_MASKED         = 4, // flat-tree leaf marker: decoded in the SECOND pass, only the blocks that hold a docID of the bitmap in slot `src`
        F_MASKOP         = 8  // flat-tree slot operation of the mask section (runs between the two decode passes)
};

struct DevStep {
        uint8_t  op, mode, dst, src;
        uint8_t  flags, pad[3];
        uint32_t term;
        uint32_t pad2;
        double   idf;
};
static_assert(sizeof(DevStep) == 24, "DevStep layout");

struct DevQuery {
        uint32_t step_begin, nsteps;
        uint32_t tile_lo, ntiles; // tiles [tile_lo, tile_lo + ntiles)
        uint32_t item_base;       // first work item of this query
        uint32_t root_slot;
        uint32_t cand_base; // SCORED_TOPK: first candidate slot of this query
        uint32_t cand_cap;
        uint32_t gen_base;  // the query's first ticket in the step-program launch (k_exec_tiles / k_exec_docs); queries other kernels / launches run own none
        uint32_t gen_base2; // k_exec_docs, second launch (flat-tree plans on a smaller tile): the query's first ticket there
        uint32_t route;     // the path the query runs: TRN_ROUTE_* (include/trinity_b200.h), decided by plan_batch (planner.h).  A candidate-driven
                            // query's items are 32-block groups of its lead term and root_slot is the number of its necessary terms (plan_batch);
                            // a flat-tree program has the layout of flat_tree_transform
};

// ---- flat scored disjunctions (k_score_flat, score_flat.cuh)
struct FlatLeaf {
        uint32_t term; // kEmptyTerm: the query names a term this index source does not hold
        uint32_t pad;
        double   idf;
};
static_assert(sizeof(FlatLeaf) == 16, "FlatLeaf layout");
struct FlatQuery {
        uint32_t qid; // position in the batch: match_counts / theta / cand_cursor index
        uint32_t leaf_begin, nleaf;
        uint32_t tile_lo, ntiles;
        uint32_t nruns;      // top-k: ceil(ntiles / run_tiles) work items
        uint32_t cand_base, cand_cap;
        uint32_t item_base;  // scored-all: the query's first (query, tile) item in the batch-wide segment arrays
        uint32_t local_base; // scored-all: the query's first item in this kernel's own ticket space
};
struct ScoreParams {
        DevIndex         ix;
        const FlatQuery *fq;
        const FlatLeaf * leaves;
        const float *    luts; // [leaf][64]
        uint32_t         nflat, total_items, run_tiles, tile_shift;
        int              mode; // TRN_MODE_SCORED_ALL / TRN_MODE_SCORED_TOPK
        uint32_t         k;
        uint32_t *       ticket;
        unsigned long long *match_counts;
        uint32_t *          theta;
        uint32_t *          cand_cursor;
        uint2 *             cand;
        unsigned long long *seg_cursor;
        uint64_t            seg_capacity;
        uint32_t *          seg_docids;
        float *             seg_scores;
        uint64_t *          item_off;
        uint32_t *          item_cnt;
        uint32_t *          overflow;
};

// one unit of the whole-list decode kernels (decode_stream.cuh): 32 consecutive blocks of one term, laid out by the host
struct DecUnit {
        uint32_t first_entry; // index of the unit's first block in blk_last / blk_off
        uint32_t cnt;         // blocks in the unit (1..32)
        uint32_t term_start;  // 1: the unit starts the term (its first block's previous docID is 0)
        uint32_t last_n;      // documents of the unit's last block when that is the term's last (possibly short) block, else 0
        uint32_t ti;          // position of the term in the caller's term list (checksum / output row index)
        uint32_t g0;          // index of the unit's first block within its term
        uint32_t pad0, pad1;
};
static_assert(sizeof(DecUnit) == 32, "DecUnit layout");

struct ExecParams {
        DevIndex        ix;
        const DevQuery *queries;
        const DevStep * steps;
        uint32_t        nq;
        uint32_t        total_items;
        uint32_t        gen_items; // number of tickets of this launch (items of the queries it runs)
        uint32_t        gen_sel;   // k_exec_docs: 0 = tickets follow DevQuery::gen_base, 1 = gen_base2
        uint32_t        has_phrase; // some plan of the batch holds OP_PHRASE: launch the instantiation that executes it
        uint32_t        nslots; // bitmap slots per worker (CTA for k_exec_tiles, warp for k_exec_docs)
        uint32_t        stage_bytes; // per-warp staging bytes of k_exec_tiles (codec dependent)
        uint32_t        docs_stage_bytes; // per-warp staging bytes of k_exec_docs (1 or 2 gather buffers)
        uint32_t        exec_shift; // log2 of the docID tile of THIS launch
        int             mode;   // TRN_MODE_*
        uint32_t        k;
        uint32_t *      ticket; // work-item dispenser
        // docs-only / scored-all outputs: segments allocated by atomicAdd on seg_cursor
        unsigned long long *seg_cursor;
        uint64_t            seg_capacity;
        uint32_t *          seg_docids;
        float *             seg_scores;
        uint64_t *          item_off; // per work item: offset of its segment
        uint32_t *          item_cnt; // per work item: number of matches (compact results: 32-bit words of its segment)
        // compact DocumentsOnly results (TRN_MODE_DOCS_COMPACT): a tile's matches leave the device as the tile's bitmap, as 16-bit offsets
        // from the tile's first docID, or as plain docIDs — whichever is smallest
        uint32_t *          item_desc;   // null unless compact: per work item, matches | encoding << 30 (trn_result::item_desc)
        unsigned long long *word_counts; // per query: words of its segments
        // top-k
        unsigned long long *match_counts; // per query
        uint32_t *          theta;        // per query: lower bound (float bits) of the k-th best score
        uint32_t *          cand_cursor;  // per query
        uint2 *             cand;         // (score bits, docid)
        uint32_t *          overflow;     // set to 1 if seg_capacity was exceeded
};

// device-side GOOGLE encoder (encode_google.cuh)
struct EncParams {
        const unsigned long long *term_begin; // nterms + 1: first posting of every term in docids[] / freqs[]
        const unsigned long long *blk_begin;  // nterms + 1: first block of every term in the flat block numbering
        uint32_t                  nterms;
        uint64_t                  nblocks;
        const uint32_t *          docids;
        const uint32_t *          freqs;
        const uint32_t *          positions; // every document's hits, concatenated in posting order; nullptr: positions 1..freq (what the synthetic builders write without hits)
        const unsigned long long *hit_begin; // exclusive scan of freqs (with positions)
        uint32_t                  block_docs, skiplist_step, phase0; // phase0: blocks committed so far by the session, modulo skiplist_step
        uint32_t *                bsz;       // bytes of every block (header included)
        uint32_t *                bterm;     // term of every block
        const unsigned long long *boff;      // exclusive scan of bsz
        const unsigned long long *term_off;  // nterms + 1: chunk offsets in out[]
        uint8_t *                 out;
        uint32_t *                error;     // != 0: an input the reference encoder throws on (docIDs not ascending / 0, positions decreasing or 0)
};

} // namespace trn
