/*
 * trinity_b200 — C ABI of the GPU-native (H100, sm_90a) execution engine for Trinity's inverted-index hot path
 * (postings-block decode -> docset AND/OR/NOT -> per-doc BM25 -> top-k).
 *
 * This is the drop-in boundary: plain pointers and sizes, int return codes (0 = ok, <0 = error; the message is
 * available from trn_last_error()), no exceptions cross it, no torch types.  Each entry point cites the
 * reference interface it stands in for (file:line under the reference tree); INTEGRATION.md shows the
 * reference-side C++ binding (GpuAccessProxy / GpuDocsSetSpan) a Trinity maintainer would add on top.
 */
#ifndef TRINITY_B200_H
#define TRINITY_B200_H
#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define TRN_OK 0
#define TRN_ERR_ARG (-1)
#define TRN_ERR_CUDA (-2)
#define TRN_ERR_FORMAT (-3)
#define TRN_ERR_STATE (-4)
#define TRN_ERR_PARSE (-5)
#define TRN_ERR_CAPACITY (-6)
#define TRN_ERR_UNSUPPORTED (-7) /* a plan uses something this engine does not execute (yet): never a silent wrong answer */

/* codec identifiers == AccessProxy::codec_identifier() "GOOGLE" / "LUCENE" (codecs.h:312, google_codec.h:101, lucene_codec.h:213) */
#define TRN_CODEC_GOOGLE 0
#define TRN_CODEC_LUCENE 1

/* == Trinity::term_index_ctx {documents, indexChunk{offset,len}} (codecs.h:17-55) */
typedef struct trn_term {
        uint32_t documents;
        uint32_t chunk_off;
        uint32_t chunk_len;
} trn_term;

/* ------------------------------------------------------------------------------------------------ index build
 * == Codecs::IndexSession + Codecs::Encoder (codecs.h:66-200; google_codec.cpp:9-176; lucene_codec.cpp:163-388).
 * Host code; produces bytes identical to the reference encoders'. */
typedef struct trn_builder trn_builder;
int  trn_builder_create(int codec, trn_builder **out);
void trn_builder_destroy(trn_builder *);
/* streaming interface == Encoder::{begin_term,begin_document,new_hit,end_document,end_term} */
int trn_builder_begin_term(trn_builder *);
int trn_builder_begin_document(trn_builder *, uint32_t docid);
int trn_builder_new_hit(trn_builder *, uint32_t position, const uint8_t *payload, uint8_t payload_len);
int trn_builder_end_document(trn_builder *);
int trn_builder_end_term(trn_builder *, trn_term *out);
/* whole-term convenience: positions = absolute positions of every hit, concatenated (sum(freqs) entries); NULL => 1..freq */
int trn_builder_add_term(trn_builder *, const uint32_t *docids, const uint32_t *freqs, uint32_t n, const uint32_t *positions, trn_term *out);
/* Google only: the encoder's skiplist countdown is session state that survives end_term (google_codec.h:57) */
int trn_builder_set_google_skiplist_countdown(trn_builder *, uint32_t countdown);
/* Google only, decode sweep only: documents per block / blocks per skiplist entry (the reference format is 32 / 8) */
int trn_builder_set_google_block(trn_builder *, uint32_t block_docs, uint32_t skiplist_step);
/* buffers stay owned by the builder */
int trn_builder_index(trn_builder *, const uint8_t **index, uint64_t *nbytes);
int trn_builder_hits(trn_builder *, const uint8_t **hits, uint64_t *nbytes); /* Lucene hits.data; 0 bytes for Google */
const char *trn_builder_last_error(trn_builder *);

/* ------------------------------------------------------------------------------------------------ synthetic index
 * The BASELINE.md workload generator (SURVEY.md 8d): V terms, df_r = max(min_df, floor(0.5*N/r)), geometric docID gaps
 * from splitmix64(seed ^ r), freq = 1 + min(7, Geom(1/2)), positions cumulative 1+u(1..16).  Multi-threaded over terms;
 * byte-identical to feeding the same postings to one reference encoder term after term. */
typedef struct trn_synth trn_synth;
int  trn_synth_build(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, trn_synth **out);
/* docID-range shard [doc_lo, doc_hi] of the same index (global docIDs kept): one IndexSource of a docID-partitioned collection */
int  trn_synth_build_shard(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, uint32_t doc_lo,
                           uint32_t doc_hi, trn_synth **out);
/* the same with the two compile-time constants of the GOOGLE format (google_codec.h:17-20: N = 32, SKIPLIST_STEP = 8) as parameters —
 * ONLY for the decode sweep of BASELINE.json configs[4]: other values are not the reference's on-disk format, trn_upload_index detects the
 * block size and the exec entry points refuse such an index (TRN_ERR_UNSUPPORTED); trn_decode_terms handles 1..128 documents per block */
int  trn_synth_build_ex(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, uint32_t doc_lo,
                        uint32_t doc_hi, uint32_t google_block_docs, uint32_t google_skiplist_step, trn_synth **out);
void trn_synth_destroy(trn_synth *);
int  trn_synth_index(trn_synth *, const uint8_t **index, uint64_t *nbytes);
int  trn_synth_hits(trn_synth *, const uint8_t **hits, uint64_t *nbytes);
int  trn_synth_terms(trn_synth *, const trn_term **terms, uint32_t *nterms);
uint64_t trn_synth_sum_hits(trn_synth *);
/* regenerate the raw postings of term rank r (1-based) — used by tests to feed the reference encoder the same input */
int trn_synth_postings(uint32_t ndocs, uint32_t rank, uint32_t min_df, uint64_t seed, uint32_t *docids, uint32_t *freqs, uint32_t cap, uint32_t *n);
int trn_synth_positions(uint32_t ndocs, uint32_t rank, uint32_t min_df, uint64_t seed, uint32_t *positions, uint64_t cap, uint64_t *n);

/* Load-time block directory of one term (host; what trn_upload_index builds for every term): last docID and payload byte
 * offset of each block (+ one sentinel entry).  == the skiplist parse of Decoder::init (google_codec.cpp:936-983,
 * lucene_codec.cpp:877-932) extended to every block.  Exposed for tests / tooling. */
int trn_directory_probe(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *term, uint32_t *blk_last, uint32_t *blk_off, uint32_t cap,
                        uint32_t *nblocks, uint32_t *first_doc, char *err, size_t errcap);

/* The kernels' docID -> block lookup run on the host over one term's directory (the same code, csrc/dirlookup.h): blocks[i] = first block
 * of the term whose last docID is >= docids[i] (nblocks if none) == skiplist_search + header hops of Decoder::advance
 * (google_codec.cpp:464-495,821-934; lucene_codec.cpp:596-656).  *tf_shift = log2 of the term's table granularity (32: no table). */
int trn_directory_lookup(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *term, const uint32_t *docids, uint32_t n, uint32_t *blocks,
                         uint32_t *tf_shift, uint32_t *tf_entries, char *err, size_t errcap);

/* Size of the whole load-time directory trn_upload_index would build (host only, no GPU): block entries (8 B per block + sentinel),
 * the sparse docID -> block tables and the per-term records.  It is O(blocks + terms) — a term's table never has more entries than
 * the term has blocks, and covers only the docID range the term occupies in THIS index source. */
int trn_directory_stats(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, int threads, uint64_t *directory_bytes,
                        uint64_t *total_blocks, uint64_t *table_entries, char *err, size_t errcap);

/* ------------------------------------------------------------------------------------------------ segment directories
 * Host half of SegmentIndexSource (segment_index_source.cpp:5-186): opens a segment directory written by Trinity's
 * SegmentIndexSession::commit() (indexer.cpp:241-300: `index`, `terms.data`, `id`, `updated_documents.ids`) and exposes what
 * trn_upload_index / trn_set_masked_documents need.  Buffers stay owned by the trn_segment. */
typedef struct trn_segment trn_segment;
int  trn_segment_open(const char *dir, trn_segment **out, char *err, size_t errcap);
void trn_segment_close(trn_segment *);
/* codec + IndexSource::field_statistics (index_source.h:44-53) restored from the `id` file */
int trn_segment_info(trn_segment *, int *codec, uint32_t *nterms, uint64_t *index_bytes, uint64_t *sum_term_hits, uint32_t *total_terms,
                     uint64_t *sum_terms_docs, uint32_t *docs_cnt, uint64_t *nmasked);
int trn_segment_index(trn_segment *, const uint8_t **index, uint64_t *nbytes);
/* the terms dictionary (terms.data, terms.cpp:125-170), in dictionary order: names[i] <-> terms[i] */
int trn_segment_terms(trn_segment *, const trn_term **terms, const char *const **names, uint32_t *nterms);
/* docIDs recorded in updated_documents.ids: what THIS segment masks in OLDER segments (index_source.h:191-238) */
int trn_segment_masked(trn_segment *, const uint32_t **docids, uint64_t *n);

/* ------------------------------------------------------------------------------------------------ query plans
 * A query is a flat node array == the reference's compiled exec_node tree (compilation_ctx.h:8-30 ENT::*) after
 * queryexec_ctx::build_iterator's flattening (exec.cpp:253-449):
 *   TERM      -> PostingsListIterator          AND -> Conjuction / ConjuctionAllPLI
 *   OR        -> Disjunction / DisjunctionAllPLI
 *   NOT       -> Filter(req = child 0, excl = child 1)           (docset_iterators.cpp:652-677)
 *   OPTIONAL  -> Optional(main = child 0, opt = child 1)         (docset_iterators.h:174-206)
 *   SOME      -> DisjunctionSome(children, min = term)           (docset_iterators.cpp:679-811; ast_node::Type::MatchSome): matches the
 *                documents at least `min` children match, scores the sum of the children that match (docset_iterators_scorers.cpp:38-56)
 *   PHRASE    -> Phrase(terms in order)   (docset_iterators.cpp:66-224): children are TERM nodes in phrase order; a document
 *                matches when some position p of the first term has term k at p+k for every k; scores score(matchCnt, Σ idf)
 * children of node i are nodes[first_child .. first_child + nchildren). */
#define TRN_NODE_TERM 0
#define TRN_NODE_AND 1
#define TRN_NODE_OR 2
#define TRN_NODE_NOT 3
#define TRN_NODE_OPTIONAL 4
#define TRN_NODE_SOME 5
#define TRN_NODE_PHRASE 6 /* executed on the GOOGLE codec (inline hits, google_codec.cpp:533-594) and, once trn_upload_hits has handed over hits.data, on the
                           * LUCENE codec (lucene_codec.cpp:767-856); a LUCENE source without its hits rejects phrase plans (TRN_ERR_UNSUPPORTED, never a silent answer) */

typedef struct trn_qnode {
        uint8_t  kind;
        uint8_t  nchildren;
        uint16_t first_child;
        uint32_t term;  /* TERM: index into the uploaded terms table; SOME: min-should-match (1..15) */
        double   weight; /* TERM: BM25 idf weight == ScorerWeight::idf (similarity.h:190-222); ignored in docs-only mode */
} trn_qnode;

typedef struct trn_query {
        const trn_qnode *nodes;
        uint32_t         nnodes;
        uint32_t         root;
} trn_query;

/* Host-side front-end for the operator subset of the reference query language (queries.cpp:11-27,150-218,477-520:
 * AND / OR / '|' / NOT / '-' / parentheses / juxtaposition = AND; OR binds tighter than AND/NOT; left-assoc), followed by the
 * same flattening build_iterator applies.  term names are resolved through `names` (nterms C strings).
 * Writes at most cap nodes; *nnodes receives the count, *root the root index. */
int trn_parse_query(const char *text, const char *const *names, uint32_t nterms, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root,
                    char *err, size_t errcap);
/* The same with an explicit terms dictionary (== IndexSource::resolve_term_ctx's lookup, index_source.h:118), built once per vocabulary
 * and owned by the caller.  trn_parse_query above rebuilds its map on every call and caches nothing. */
typedef struct trn_dict trn_dict;
int  trn_dict_create(const char *const *names, uint32_t nterms, trn_dict **out);
void trn_dict_destroy(trn_dict *);
int  trn_parse_query_dict(const char *text, const trn_dict *dict, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root, char *err, size_t errcap);

/* The boolean function of a query tree over its distinct (non-empty) terms, as the planner of the candidate-driven path tabulates
 * it (DocumentsOnly; == which term combinations DocsSetIterators::Conjuction / Disjunction / Filter / Optional / DisjunctionSome
 * accept): terms[j] = j-th distinct term (<= 8, else TRN_ERR_ARG); bit a of table[] (256 bits) = value of the query when exactly
 * the terms whose bit is set in a are on the document; *necessary = mask of the terms every match holds.  Host-only (tests, tooling). */
int trn_query_truth_table(const trn_qnode *nodes, uint32_t nnodes, uint32_t root, uint32_t *terms, uint32_t *nterms, uint32_t *table, uint32_t *necessary);

/* Host-only view of the plan compiler (tests, tooling): the step program trn_exec_batch would run for one query on the bitmap paths —
 * == the iterator tree build_iterator/build_span would have built (exec.cpp:253-505), flattened into slot operations.  op: 0 LEAF
 * (decode term into / against slot dst with mode), 1 SLOT (combine slot src into dst), 2 CLEAR, 3 LEAFSCORE (second scoring pass of
 * `term` where slot src has the document), 4 COUNT_ADD / 5 COUNT_GE (MatchSome counters); mode: 0 SET 1 OR 2 AND 3 ANDNOT 4 NONE;
 * flags: 1 = the leaf scores where it matches, 2 = stop when dst becomes empty.  Needs no GPU.
 * scored: 0 = DocumentsOnly program, 1 = scored program, 2 = DocumentsOnly program in its flat-tree form (every leaf owns a bitmap announced
 * by a leading [LEAF, mode NONE, dst = leaf slot] marker and filled by one flat pass over the tile; slot operations only afterwards). */
typedef struct trn_debug_step {
        uint8_t  op, mode, dst, src, flags, pad[3];
        uint32_t term;
        uint32_t pad2;
        double   idf;
} trn_debug_step;
/* the kernels' position cursors (csrc/hitcursor.h) run on the host over one term: positions of the listed documents (counts[i] each), for
 * the CPU tests; `hits` = hits.data (LUCENE), ignored for GOOGLE */
int trn_debug_positions(int codec, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hits_bytes, const trn_term *term, const uint32_t *docids, uint32_t n,
                        uint32_t *counts, uint32_t *positions, uint64_t cap, uint64_t *total, char *err, size_t errcap);
int trn_debug_compile(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, const trn_qnode *nodes, uint32_t nnodes, uint32_t root,
                      int scored, trn_debug_step *out, uint32_t cap, uint32_t *nsteps, uint32_t *root_slot, uint32_t *nslots, char *err, size_t errcap);

/* BM25 weight of one term == IndexSourcesCollectionBM25Scorer::Scorer::idf evaluated in float (similarity.h:179-181) */
double trn_bm25_idf(uint32_t doc_freq, uint64_t docs_cnt);
/* == Scorer::score(id, freq, weight) (similarity.h:228-235): float(idf * float(freq) / double(freq + 1.2f)) */
float trn_bm25_score(double idf, uint16_t freq);

/* ------------------------------------------------------------------------------------------------ engine
 * trn_ctx == one device-resident IndexSource (index_source.h:18-155) + its AccessProxy (codecs.h:290-317). */
typedef struct trn_ctx trn_ctx;

int         trn_create(int device, trn_ctx **out);
void        trn_destroy(trn_ctx *);
const char *trn_last_error(trn_ctx *);
/* run on this cudaStream_t (default: the legacy default stream). Lets callers time with their own events. */
int trn_set_stream(trn_ctx *, void *cuda_stream);

/* == AccessProxy(basePath, indexPtr) + Decoder::init for every term (google_codec.cpp:936-983, lucene_codec.cpp:877-932):
 * copies the raw, unmodified index bytes to HBM and builds the block directory.  max_docid = upper bound of the docID space; 0 = take
 * the largest docID found in the postings (a segment directory does not record it). */
int trn_upload_index(trn_ctx *, int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid);

/* == masked_documents_registry (docidupdates.h:90-190): documents deleted/updated by newer index sources.  The reference tests every
 * match against it in the exec Handlers (exec.cpp:1108-1116, `if (!maskedDocumentsRegistry->test(id)) consider(...)`); here the docIDs are
 * kept as a device bitmap that is AND-NOTed into every tile's result before emission / top-k.  n == 0 clears the registry; docIDs
 * above max_docid are ignored (a newer source may mask documents this source never held). */
int trn_set_masked_documents(trn_ctx *, const uint32_t *docids, uint64_t n);

typedef struct trn_index_info {
        int      codec;
        uint32_t nterms, max_docid, tile_docs, ntiles, block_docs;
        uint64_t index_bytes, directory_bytes, total_blocks, total_postings;
} trn_index_info;
int trn_index_info_get(trn_ctx *, trn_index_info *out);

/* LUCENE positions == Lucene AccessProxy::hitsDataPtr (lucene_codec.h:204-218): hits.data of the index uploaded before, for phrase plans
 * (TRN_NODE_PHRASE).  `index` = the bytes trn_upload_index received (read again on the host to lay out the hits directory).  The GOOGLE
 * codec keeps its hits inline and needs no such call. */
int trn_upload_hits(trn_ctx *, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hits_bytes);

/* execution modes == ExecFlags (exec.h:12-43) + where top-k lives */
#define TRN_MODE_DOCS_ONLY 0    /* ExecFlags::DocumentsOnly: matched docIDs ascending == consider(docid_t) stream        */
#define TRN_MODE_SCORED_ALL 1   /* ExecFlags::AccumulatedScoreScheme: every (docID, score) ascending == consider(id,score) */
#define TRN_MODE_SCORED_TOPK 2  /* AccumulatedScoreScheme + the application's top-k sink fused on device                 */
#define TRN_MODE_DOCS_COMPACT 3 /* DocumentsOnly, the same consider(docid_t) stream in a compact encoding (below): the matched docIDs of a
                                 * large batch are what the host link carries, so dense result tiles travel as bitmaps and sparse ones as
                                 * 16-bit offsets; trn_result_for_each / trn_result_decode replay them                                    */

/* Result of a batch. Host pointers are pinned buffers owned by the ctx, valid until the next exec call.
 * DOCS_ONLY / SCORED_ALL: query q owns [offsets[q], offsets[q+1]) of docids (ascending) (+ scores).
 * SCORED_TOPK: query q owns [offsets[q], offsets[q+1]) with at most k entries ordered by (score desc, docID asc);
 * match_counts[q] = total number of matching documents. */
typedef struct trn_result {
        uint32_t        nq;
        uint64_t        total;
        const uint64_t *offsets;
        const uint32_t *docids;
        const float *   scores;
        const uint64_t *match_counts;
        uint64_t        postings_scanned; /* sum over queries of sum over leaf terms of term.documents (full-scan accounting, SURVEY 8d) */
        uint64_t        index_bytes_touched; /* sum over queries of sum over leaf terms of chunk_len (algorithmic bytes, SURVEY 8d)        */
        uint32_t        kernel_launches;
        float           device_ms; /* CUDA-event time of the device part of this call (plan H2D + all kernels) */
        float           exec_kernel_ms; /* CUDA-event time of the fused k_exec_tiles launch alone (roofline denominator) */
        /* TRN_MODE_DOCS_COMPACT (null / 0 otherwise): `docids` is null; query q owns the 32-bit words [offsets[q], offsets[q+1]) of `words`,
         * made of the segments of its work items qitems[q].item_base .. + nitems, in ascending docID order.  Segment i holds
         * item_desc[i] & 0x3fffffff documents in the encoding item_desc[i] >> 30 and takes that many words:
         *   TRN_ENC_U32    docIDs, one per word                                                              (count words)
         *   TRN_ENC_U16    offsets from the first docID of the item's tile, two per word, low half first      ((count + 1) / 2 words)
         *   TRN_ENC_BITMAP the tile's bitmap, bit b of word w = docID tile_first + 32 w + b                   (2^tile_shift / 32 words)
         *   TRN_ENC_U8B    the tile in 256-docID buckets: 2^tile_shift / 256 count bytes (documents of every bucket, < 256 each), then one
         *                  offset byte per document (docID = tile_first + 256 bucket + offset), zero-padded to a word   ((buckets + count + 3) / 4 words)
         * the tile of item j of query q starts at docID (qitems[q].tile_lo + j) << qitems[q].tile_shift (U16 / U8B / BITMAP segments only). */
        const uint32_t *         words;
        uint64_t                 total_words;
        const uint32_t *         item_desc;
        const struct trn_qitems *qitems;
} trn_result;
#define TRN_ENC_U32 0u
#define TRN_ENC_U16 1u
#define TRN_ENC_BITMAP 2u
#define TRN_ENC_U8B 3u
typedef struct trn_qitems {
        uint32_t item_base, nitems;
        uint32_t tile_lo, tile_shift;
} trn_qitems;
/* Replay of query q's matches, ascending, exactly once each == the MatchesProxy::process / consider(docid_t) stream (docset_spans.h:14-21,
 * matches.h:149-171); works for DOCS_ONLY and DOCS_COMPACT results.  `fn` returning non-zero stops the replay (aborted_search_exception). */
typedef int (*trn_consider_fn)(void *ctx, uint32_t docid);
int trn_result_for_each(const trn_result *r, uint32_t q, trn_consider_fn fn, void *ctx);
/* query q's matched docIDs into out[0..cap); *n = their number (== match_counts[q]); TRN_ERR_CAPACITY if cap is too small */
int trn_result_decode(const trn_result *r, uint32_t q, uint32_t *out, uint64_t cap, uint64_t *n);

/* == exec_query(query, IndexSource*, masked_documents_registry*, MatchedIndexDocumentsFilter*, ..., flags, scorer) (exec.h:50-52),
 * batched (SURVEY 8b: gpu_exec_queries).  H2D of the plans and D2H of the results are part of the call. */
int trn_exec_batch(trn_ctx *, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out);

/* Host-side wall-clock breakdown of the last trn_exec_batch / trn_exec_batch_device call of this ctx (milliseconds): where a rank's
 * end-to-end time goes when several ranks share one host (bench.py prints it per rank). */
typedef struct trn_timings {
        float host_compile_ms; /* plan compilation (== build_iterator + build_span per query, exec.cpp:253-505) */
        float enqueue_ms;      /* buffer sizing, plan H2D and kernel launches (asynchronous enqueue) */
        float chunk_wait_ms;   /* pipelined call: blocked until a chunk's kernels finished (its counts are needed to size the result copy) */
        float final_wait_ms;   /* blocked at the end: last kernels + result D2H */
        float kernel_ms;       /* CUDA-event time of the fused exec kernels (device) */
        float total_ms;        /* the whole call */
        float chunks;          /* pipelined call: chunks the batch was split into (sized by the postings it references); 1 = single call */
} trn_timings;
int trn_last_timings(trn_ctx *, trn_timings *out);
/* Host-only view of the pipeline planner (tests, tooling): the launches trn_exec_batch would split a DocumentsOnly / SCORED_ALL batch into, from
 * what it knows before the first launch — referenced postings and TERM nodes of the batch, the knobs (TRN_PIPELINE_CHUNKS, TRN_CHUNK_POSTINGS,
 * TRN_CHUNK_RULE, TRN_TAPER_CHUNKS, TRN_CHUNK_TAIL_US, TRN_CHUNK_TAIL_TREE_US) and the previous batch's result bytes / postings / shape.
 * sizes[] receives the queries per launch, *n their number, *single_call whether the batch takes the one-call form. */
int trn_debug_chunk_plan(uint32_t nq, int topk, uint64_t est_postings, uint64_t leaves, uint32_t max_chunks, uint64_t chunk_postings, int rule_sqrt, int taper,
                         double tail_ms, double tail_tree_ms, uint64_t hint_bytes, uint64_t hint_postings, int hint_same_shape, uint32_t *sizes, uint32_t cap,
                         uint32_t *n, int *single_call);

/* Debug view (tests, tooling): the path the host chose for every query of the last trn_exec_batch / trn_exec_batch_device call, one
 * TRN_ROUTE_* code per query into out[0..cap); *n = the batch's query count (TRN_ERR_CAPACITY if cap is smaller; 0 after a failed call).
 * DocumentsOnly plans run in k_exec_docs as a step program, a flat AND / OR of terms (GOOGLE), the candidate-driven conjunction (GOOGLE)
 * or a flat tree (GOOGLE); scored plans run in k_score_flat (LUCENE flat OR / single term) or k_exec_tiles.  A flat AND needs one docset
 * slot per operand: it is reported as a step program when its launch has fewer slots (the effective limit is min(16, slots of the launch);
 * conjunctions of <= 3 terms raise the slot count themselves).  The codes are plan-level: a flat AND whose rarest operand is sparse in
 * a tile still runs that tile as a step program, and such per-tile choices are not visible here. */
#define TRN_ROUTE_STEPS 0        /* DocumentsOnly: step program of k_exec_docs                       */
#define TRN_ROUTE_FLAT_AND 1     /* DocumentsOnly: flat conjunction of terms (GOOGLE)                */
#define TRN_ROUTE_FLAT_OR 2      /* DocumentsOnly: flat disjunction of terms (GOOGLE)                */
#define TRN_ROUTE_CANDIDATE 3    /* DocumentsOnly: candidate-driven evaluation (GOOGLE)              */
#define TRN_ROUTE_SCORE_FLAT 4   /* scored: k_score_flat (LUCENE)                                    */
#define TRN_ROUTE_FLAT_TREE 5    /* DocumentsOnly: flat-tree form of the step program (GOOGLE)       */
#define TRN_ROUTE_EXEC_TILES 6   /* scored: step program of k_exec_tiles                             */
int trn_debug_last_routes(trn_ctx *, uint8_t *out, uint32_t cap, uint32_t *n);
/* Host-only view of the same decision (tests, tooling; no GPU needed): plans a batch as trn_exec_batch would on a context that trn_create
 * made with this environment and that holds this index (trn_upload_index's arguments), without executing it.  routes[0..nq) receives the
 * TRN_ROUTE_* of every query, nslots[0] the docset slots of the step-program launch (k_exec_docs / k_exec_tiles), nslots[1] those of the
 * flat-tree launch of k_exec_docs.  LUCENE phrase plans are refused as on a context without trn_upload_hits. */
int trn_debug_plan(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid, const trn_query *queries,
                   uint32_t nq, int mode, uint32_t k, uint8_t *routes, uint32_t *nslots, char *err, size_t errcap);

/* Split form used by bench.py / multi-GPU: run on device only, results stay in HBM ... */
int trn_exec_batch_device(trn_ctx *, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out_counts_only);
/* ... device pointers of the last SCORED_TOPK run: nq*k u32 docids, nq*k f32 scores (unused slots: docid 0, score -1.0; real scores are >= 0), nq u32 counts */
int trn_last_topk_device(trn_ctx *, void **docids, void **scores, void **counts);
/* merge `nshards` gathered top-k lists (layout [shard][nq][k]) into one; the one exchange step of the multi-GPU path (SURVEY 8e).
 * All pointers are device pointers; docid_base[shard] is added to the docids of that shard (0 if docIDs are already global). */
int trn_merge_topk(trn_ctx *, const void *docids, const void *scores, uint32_t nshards, uint32_t nq, uint32_t k, void *out_docids, void *out_scores);
/* copy the last device results to the pinned host buffers (the D2H leg) and fill `out` */
int trn_fetch_results(trn_ctx *, trn_result *out);

/* Decode microbench / parity probe == PostingsListIterator::next() over whole lists (google_codec.cpp:777-819, lucene_codec.cpp:568-594).
 * materialise != 0: writes docids/freqs (host pointers, sum(documents) entries, terms concatenated in the given order);
 * materialise == 0: fused checksum only (sum of docids and sum of freqs per term into sums[2*i], sums[2*i+1]). */
int trn_decode_terms(trn_ctx *, const uint32_t *term_ids, uint32_t nterms, int materialise, uint32_t *docids, uint32_t *freqs, uint64_t *sums,
                     float *device_ms);

/* GPU-side Encoder, GOOGLE layout == Codecs::Google::Encoder begin_term / begin_document / new_hit / end_document / end_term
 * (google_codec.cpp:9-176; google_codec.h:17-20 N = 32, SKIPLIST_STEP = 8) for hits without payloads: the index is BUILT on the device
 * (SURVEY.md 8(f) row 4), byte for byte what the reference encoder writes for the same postings.  All pointers are HOST pointers:
 *   term_begin[nterms + 1]  first posting of every term in docids[] / freqs[] (term i holds [term_begin[i], term_begin[i+1]))
 *   docids[], freqs[]       ascending docIDs > 0 per term; freqs[i] = hits of posting i
 *   positions[]             the hits of all postings, concatenated in posting order (sum(freqs) entries, in 1..16383 = below Limits::MaxPosition, non-decreasing per document);
 *                           NULL = positions 1..freq (what an index built without positions carries)
 *   block_docs / skiplist_step  the two compile-time constants of the format (32 / 8 = the reference's; other values only for the
 *                           decode sweep, BASELINE.json configs[4]); *countdown (in/out, may be NULL = a fresh session) = the encoder
 *                           session's skiplistEntryCountdown, which carries over between terms (google_codec.h:57)
 *   out[cap]                receives the chunks of the terms back to back; *out_bytes their total (also when cap is too small:
 *                           TRN_ERR_CAPACITY, nothing written); terms[nterms] the term_index_ctx tuples
 * TRN_ERR_ARG: an input the reference encoder throws on (docID 0 / not ascending, a position 0 / decreasing / >= Limits::MaxPosition).
 * *device_ms (may be NULL): the device time of the encode (kernels and the two scans), without the host<->device copies. */
int trn_encode_google(trn_ctx *, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                      uint32_t block_docs, uint32_t skiplist_step, uint32_t *countdown, uint8_t *out, uint64_t cap, uint64_t *out_bytes, trn_term *terms,
                      float *device_ms);

#ifdef __cplusplus
}
#endif
#endif
