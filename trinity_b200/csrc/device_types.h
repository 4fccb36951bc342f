// Device-side data layout shared by the host (planner.cpp, engine.cu) and kernels.cu (device).
#pragma once
#include "../../include/trinity_b200.h"
#include <cstdint>
#include <vector_types.h>

namespace trn {

struct HitTerm;

static constexpr uint32_t kEmptyTerm = 0xffffffffu;
// resident bitmaps of dense terms (DevIndex::dense): both ends of a term's bitmap aligned to 2^17 docIDs, the largest k_exec_docs tile
static constexpr uint32_t kDenseAlignShift = 17;
static constexpr uint32_t kDenseNone       = 0xffffffffu;

// run tickets of flat ANDs (BatchPlan::dense_runs, mixed_runs): a ticket {query, first tile} covers the query's tiles from `first` to the end of the
// 2^kDenseAlignShift-docID run that holds it (or to the end of the query's tiles [tile_lo, tile_lo + ntiles), whichever comes first)
__host__ __device__ inline uint32_t dense_run_end(uint32_t first, uint32_t tile_lo, uint32_t ntiles, uint32_t exec_shift) {
        const uint32_t e = (first | ((1u << (kDenseAlignShift - exec_shift)) - 1u)) + 1u, qe = tile_lo + ntiles;
        return e < qe ? e : qe;
}

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
        // resident docID bitmaps of dense GOOGLE terms (planner.h select_dense_terms; null when the source has none): term t's bitmap starts
        // at word dense_off[t] of `dense` (kDenseNone: no bitmap) and covers docIDs from first_doc rounded down to 2^kDenseAlignShift.
        // probe_off (null, like `dense`, when the source has neither tier): the same for the probe bitmaps (select_probe_terms), laid out
        // behind the dense ones; it holds dense_off[t] for a term with a dense bitmap.  Only the candidate-driven conjunction probes through
        // it, and k_build_dense builds both tiers through it.
        const uint32_t *dense;
        const uint32_t *dense_off;
        const uint32_t *probe_off;
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
        F_BREAK_IF_EMPTY = 2
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
// a query's document filter (trn_doc_filter) as the kernels read it: resident docID sets laid out like DevIndex::masked.  A query
// ignores d iff masked(d) || (allow && d not in allow) || (deny && d in deny).  Only the filtered instantiations (FILT) read it.
struct DevFilter {
        const uint32_t *allow; // null: no allow set
        const uint32_t *deny;  // null: no deny set
        uint32_t        lo, hi; // the allow set's first and last docID (lo > hi: it is empty); 0, 0xffffffff without one
};
static_assert(sizeof(DevFilter) == 24, "DevFilter layout");

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
        const DevFilter *   filters; // per query of the batch (FlatQuery::qid); null: no query has a filter
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
        const uint2 *   dense_runs;  // k_exec_docs, step-program launch: tickets [0, dense_items) are the all-bitmap flat ANDs' (query, run) pairs
        uint32_t        dense_items; // (BatchPlan::dense_runs)
        const uint2 *   mixed_runs;  // ... then tickets [dense_items, dense_items + mixed_items): the flat ANDs with one decoded operand
        uint32_t        mixed_items; // (BatchPlan::mixed_runs)
        const uint32_t *cand_order;  // ... then cand_items tickets: ticket i runs gen ticket cand_order[i] (candidate-driven groups, run-major);
        uint32_t        cand_items;  // the gen tickets follow, and skip those of candidate-driven queries when cand_items != 0
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
        const DevFilter *   filters;      // per query; null: no query of the batch has a filter (the unfiltered instantiations run)
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
// the hits' payloads, beside positions[] (the encoders' payload instantiations only: the parameters of the others keep their layout)
struct EncPayloads {
        const uint8_t *           plens;    // per hit: payload bytes 0..8 (null: no payloads)
        const unsigned long long *payloads; // per hit: the payload in the low plens[] bytes, memory order
};
struct EncPayloadParams : EncParams {
        EncPayloads pay;
};

// device-side LUCENE encoder (encode_lucene.cuh).  A term's doc units are its full 128-document blocks followed by its tail (the
// documents % 128 varbyte pairs, possibly none); its hit units are its full 128-hit blocks followed by its hit tail.  Every term has
// at least one unit of each kind, so a unit's term is the last term whose first unit is <= it.
struct EncLuceneParams {
        const unsigned long long *term_begin;  // nterms + 1: first posting of every term in docids[] / freqs[]
        const unsigned long long *dunit_begin; // nterms + 1: first doc unit of every term
        const unsigned long long *hunit_begin; // nterms + 1: first hit unit of every term
        uint32_t                  nterms;
        uint64_t                  ndunits, nhunits;
        const uint32_t *          docids;
        const uint32_t *          freqs;
        const uint32_t *          positions; // every document's hits, concatenated in posting order; nullptr: positions 1..freq
        const unsigned long long *hit_begin; // nposts + 1: exclusive scan of freqs
        uint32_t *                dsz, *hsz;     // bytes of every doc / hit unit
        uint32_t *                dterm, *hterm; // term of every doc / hit unit
        const unsigned long long *doff, *hoff;   // exclusive scans of dsz / hsz (hoff is the unit's offset in hits_out)
        const unsigned long long *term_off;      // nterms + 1: chunk offsets in index_out
        uint8_t *                 index_out;
        uint8_t *                 hits_out;
        uint32_t *                error; // != 0: docIDs not ascending / 0, positions decreasing / 0 / >= Limits::MaxPosition
};
struct EncLucenePayloadParams : EncLuceneParams {
        EncPayloads pay;
};

// ---- the default exec mode (TRN_MODE_MATCHED_TERMS): which query terms a match holds (collect.cuh; planner.cpp plan_collect)
static constexpr uint32_t kCollectMaxTerms   = 32; // distinct terms of a query: one u32 mask per match
static constexpr uint32_t kCollectMaxPhrases = 32; // phrase nodes of a query: one ballot
static constexpr uint32_t kCollectMaxStack   = 32; // operands pending while the post-order program runs
enum CollectOpKind : uint8_t { CO_TERM = 0, CO_AND = 1, CO_OR = 2, CO_NOT = 3, CO_OPTIONAL = 4, CO_SOME = 5, CO_PHRASE = 6 };
struct CollectOp { // one node of the post-order collect program
        uint8_t  kind, nchildren;
        uint16_t min; // CO_SOME: min-should-match
        uint32_t arg; // CO_TERM: bit of the term in the query's table (kEmptyTerm: a term the source does not hold); CO_PHRASE: phrase index
};
struct CollectPhrase {
        uint32_t arg_begin; // first OP_ARG step of its term ids (phrase.cuh phrase_arg), in CollectPlan::args
        uint32_t k;         // terms of the phrase
        uint32_t mask;      // its terms' bits in the query's table
        uint32_t pad;
};
struct CollectQuery {
        uint32_t term_begin, nterms;     // the query's distinct terms, ascending term index (bit j = terms[term_begin + j])
        uint32_t phrase_begin, nphrases; // its phrase nodes
        uint32_t prog_begin, nprog;      // its post-order program
};
static_assert(sizeof(trn_hit) == 16, "trn_hit: payload, pos, payload_len, 5 padding bytes");
struct CollectParams {
        DevIndex             ix;
        const CollectQuery * queries;
        const uint32_t *     terms;
        const CollectPhrase *phrases;
        const DevStep *      args;
        const CollectOp *    prog;
        const uint64_t *     q_offsets; // nq + 1: the matches of query q are [q_offsets[q], q_offsets[q + 1]) of docids
        const uint32_t *     docids;
        uint32_t             nq;
        uint64_t             m0, m1;   // the launch's matches (the count kernel: the whole batch; the write kernel: one chunk)
        uint32_t *           mask;     // per match of the batch: the matched terms
        uint32_t *           nterms;   // ... their number
        uint32_t *           nhits;    // ... and the sum of their freqs
        const unsigned long long *term_scan, *hit_scan; // exclusive scans of nterms / nhits over the batch
        uint64_t             term_base, hit_base;        // the chunk's first term / hit: where out_terms ... / out_hits start
        uint64_t *           term_offsets; // per match of the chunk: its first term (global)
        uint32_t *           out_terms;    // per term of the chunk
        uint32_t *           out_freqs;
        uint64_t *           hit_offsets;  // per term of the chunk: its first hit (global)
        trn_hit *            out_hits;     // per hit of the chunk
        uint32_t *           error;        // != 0: a match the collect program does not accept (a docs-pass / program disagreement)
};

// ---- query-token intersections (trn_intersect; intersect.cuh, isectplan.h)
// a warp's group bitmaps hold 2^16 bits (intersect.cuh): a request with G groups cuts the docID space into tiles of 2^16 / max(8, G rounded up
// to a power of two) documents, 2^13 .. 2^10
inline uint32_t isect_tile_shift(uint32_t ngroups) {
        uint32_t lg = 3;
        while ((1u << lg) < ngroups)
                ++lg;
        return 16u - lg;
}
struct IsectReq {
        uint32_t tok_begin, ntok;     // its known tokens: IsectParams::tok[tok_begin .. + ntok), {term, group}
        uint32_t ngroups, shift;      // groups; log2 of its docID tile (isect_tile_shift: the more groups, the smaller the tile)
        uint32_t tile_lo, ntiles;     // tiles [tile_lo, tile_lo + ntiles) of 2^shift docIDs
        uint32_t item_base;           // its first work item
        uint32_t epoch_begin;         // pass B: its first epoch (global numbering of IsectParams::epoch_start / epoch_off)
        uint32_t nepochs;             // ...
        uint32_t pad;
        uint64_t orig_mask;           // documents holding exactly this mask are not considered (0: some token is unknown)
        uint64_t slots, table_base;   // pass A: its open-addressing table of distinct masks (slots: a power of two)
};
struct IsectParams {
        DevIndex        ix;
        const IsectReq *reqs;
        const uint2 *   tok;
        uint32_t        nreq, total_items;
        uint32_t        max_masks; // distinct masks a request may have
        uint32_t *      ticket;
        uint32_t *      error; // pass A: a table overflowed; pass B: a document found no target (internal bound violated)
        // pass A
        unsigned long long *keys;      // per table slot: the mask (0: empty)
        uint32_t *          first;     // per table slot: its first docID (atomicMin)
        uint32_t *          ndist;     // per request: distinct masks inserted
        unsigned long long *tile_last; // per work item: the mask of its last considered document (0: none)
        // pass B
        const unsigned long long *carry;      // per work item: the mask of the last considered document before its tile (0: none)
        const uint32_t *          epoch_start; // per epoch: the docID of the push that starts it
        const uint32_t *          epoch_off;   // per epoch + 1: its array is entries [epoch_off[e], epoch_off[e + 1])
        const unsigned long long *snap_mask;   // per entry: the mask
        const int32_t *           snap_slot;   // per entry: its slot in counts (-1: removed later, its count is lost)
        uint32_t *                counts;      // per final antichain entry of every request
};

// ---- percolator (trn_percolator_register / trn_percolate; percplan.h, percolate.cuh)
static constexpr uint32_t kPercMaxDocLen  = 16383; // tokens of a document: positions 1 .. 16383, below Limits::MaxPosition
static constexpr uint32_t kPercShortLen   = 512;   // documents up to this many tokens run in the short launch (small shared tables, many CTAs per SM)
static constexpr uint32_t kPercMaxHash    = 16384; // slots of a document's distinct-term table (a power of two >= 2 x its length, at most this)
static constexpr uint32_t kPercSortCap    = 4096;  // a document with at most this many matches sorts its ids in shared memory; more: a bitmap
static constexpr uint32_t kPercStack      = 64;    // evaluation stack of a query program: one bit per pending operand, in one 64-bit register
// slots of the distinct-term table of a document of L tokens (at least one more than its distinct terms)
__host__ __device__ inline uint32_t perc_hash_slots(uint32_t L) {
        uint32_t H = 32;
        while (H < 2u * L && H < kPercMaxHash)
                H <<= 1;
        return H;
}
enum : uint8_t { PERC_TERM, PERC_PHRASE, PERC_CONST, PERC_AND, PERC_OR, PERC_NOT, PERC_OPT, PERC_SOME };
// one post-order operation of a query program.  TERM: the term is on the document.  PHRASE: the n terms phrase_terms[term .. + n) stand at
// consecutive positions; arg = the index of its cheapest term (the one whose positions are tried).  CONST: the value `term`.  AND / OR /
// NOT (the first operand and none of the others) / OPT (the first operand) / SOME (at least arg >= 1 operands): of the n topmost values.
struct PercOp {
        uint8_t  op, n;
        uint16_t arg;
        uint32_t term;
};
struct PercQuery {
        uint32_t op_begin, nops;       // its program: ops[op_begin .. + nops)
        uint32_t cover_begin, ncover;  // its anchor cover, ascending term id: covers[cover_begin .. + ncover)
};
struct PercEntry {
        uint32_t query, ordinal; // an anchored query and the index of this anchor in its sorted cover
};
struct PercParams {
        // the registry
        const PercQuery *queries;
        const PercOp *   ops;
        const uint32_t * phrase_terms;
        const uint32_t * covers;
        const uint32_t * csr_off; // per term + 1: its anchored queries are csr[csr_off[t] .. csr_off[t + 1])
        const PercEntry *csr;
        const uint32_t * unanchored; // queries every document evaluates
        uint32_t         nunanchored, nterms;
        // the documents of this launch: docs[0 .. ndocs), document d = tokens[doc_off[d] .. doc_off[d + 1])
        const unsigned long long *doc_off;
        const uint32_t *          tokens;
        const uint32_t *          docs;
        uint32_t                  ndocs, max_len; // max_len: the longest document of the launch (shared token array)
        uint32_t                  max_hash;       // slots of the launch's shared distinct-term table
        // count pass
        uint32_t *          counts;     // per document: its matches
        unsigned long long *candidates; // (document, query) pairs evaluated
        // write pass
        const unsigned long long *out_off;    // per document + 1: its ids go to out[out_off[d] ..)
        uint32_t *                out;
        uint32_t *                bitmaps;    // documents with more than kPercSortCap matches: one zeroed bitmap of bitmap_words words each
        const uint32_t *          dense_slot; // ... the index of a document's bitmap
        uint32_t                  bitmap_words;
};

// ---- indexer (trn_index_documents; index_docs.cuh)
static constexpr uint32_t kIndexMaxTerms = 1u << 24; // term_order bits of a sort key
static constexpr uint32_t kIndexMaxDocs  = 1u << 26; // doc_rank bits of a sort key
// slots of IndexParams::errors: the lowest offending document ordinal / token / posting / document rank of every kind (~0: none)
// terms (transient ids 1 .. nterms, term t has id t + 1) that precede bucket b of commit()'s 32 buckets (id & 31, indexer.cpp:388): the ids
// 0 .. nterms whose residue is below b, without id 0
__host__ __device__ inline uint32_t index_bucket_start(uint32_t b, uint32_t nterms) {
        const uint32_t full = (nterms + 1u) >> 5, rem = (nterms + 1u) & 31u;
        return full * b + (b < rem ? b : rem) - (b ? 1u : 0u);
}
// the place of term t in the encode order ((t + 1) & 31, t), and the term at a place
__host__ __device__ inline uint32_t index_term_order(uint32_t t, uint32_t nterms) {
        const uint32_t u = t + 1u, b = u & 31u;
        return index_bucket_start(b, nterms) + (u >> 5) - (b ? 0u : 1u);
}
__host__ __device__ inline uint32_t index_term_at(uint32_t order, uint32_t nterms) {
        uint32_t b = 0;
        while (b < 31u && index_bucket_start(b + 1u, nterms) <= order)
                ++b;
        return (((order - index_bucket_start(b, nterms)) + (b ? 0u : 1u)) << 5 | b) - 1u;
}
enum : uint32_t { IDX_ERR_DOC0, IDX_ERR_DUP, IDX_ERR_TOKEN, IDX_ERR_POS, IDX_ERR_POS0, IDX_ERR_FREQ, IDX_ERR_DOCTERMS, IDX_ERR_PAYLEN, IDX_ERR_PAYDUP, IDX_ERR_KINDS };
struct IndexParams {
        // the batch: document d = tokens[doc_off[d] .. doc_off[d + 1]), token i at positions[i] (null: at i - doc_off[d] + 1)
        const unsigned long long *doc_off;
        const uint32_t *          tokens;
        const uint32_t *          positions;
        const uint8_t *           plens;    // per token: payload bytes 0..8; null: no payloads
        const unsigned long long *payloads; // per token: the payload in the low plens[] bytes, memory order
        uint32_t                  ndocs, nterms;
        uint64_t                  ntokens;
        const uint32_t *          rank_of;  // per document ordinal: its rank in docID order
        const uint32_t *          docid_of; // per rank: the docID
        unsigned long long *      keys;     // per token: term_order << 40 | doc_rank << 14 | position
        uint32_t *                ords;     // with payloads: per token its ordinal, the value the sort moves beside the key
        unsigned long long *      errors;   // IDX_ERR_KINDS slots
        // the postings pass over the sorted keys
        const uint32_t *          post_flag, *term_flag; // per token: opens a posting / a term
        const unsigned long long *post_scan, *term_scan; // their exclusive scans (ntokens + 1)
        unsigned long long *      post_begin; // per posting + 1: its first hit
        unsigned long long *      term_begin; // per present term + 1: its first posting
        uint32_t *                term_order; // per present term: its place in the encode order
        uint32_t *                out_docids, *out_freqs, *out_positions;
        uint8_t *                 out_plens;    // with payloads: per hit, gathered through the sorted ordinals
        unsigned long long *      out_payloads; // ... the payload, bytes past its length cleared
        uint32_t *                doc_terms;  // per rank: distinct terms (zeroed); null when nterms <= 65535 cannot exceed the limit
};

} // namespace trn
