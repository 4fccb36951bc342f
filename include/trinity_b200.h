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
 * by a leading [LEAF, mode NONE, dst = leaf slot] marker and filled by one flat pass over the tile; slot operations only afterwards).
 * Phrases compile on a GOOGLE index (7 PHRASE with mode = k, then ceil(k / 4) 8 ARG steps of term ids), as trn_debug_plan plans them. */
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
        /* resident docID bitmaps of the dense terms (GOOGLE; trn_debug_dense_terms): how many terms have one and their bytes in HBM.  Not
         * counted in directory_bytes.  0 when TRN_DENSE_BITMAPS=0, for LUCENE sources, or when the upload could not allocate them
         * (trn_last_error then says so; the upload itself succeeds). */
        uint64_t dense_terms, dense_bitmap_bytes;
        /* the probe bitmaps (GOOGLE; trn_debug_probe_terms): the second tier, which only the candidate-driven conjunction probes, for terms
         * without a dense bitmap.  How many terms have one and their bytes in HBM, beside dense_bitmap_bytes.  0 when TRN_PROBE_BITMAPS=0,
         * TRN_PROBE_BUDGET=0 or TRN_DENSE_BITMAPS=0, for LUCENE sources, or when the upload could not allocate them (trn_last_error then
         * says so; the dense tier is kept if it fits alone). */
        uint64_t probe_terms, probe_bitmap_bytes;
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
/* The same plan's run-major tickets of the all-bitmap flat ANDs (TRN_ROUTE_FLAT_AND plans whose operands all have a resident bitmap; they
 * run in front of the other tickets of the step-program launch; TRN_DENSE_RUNS=0 turns them off).  qtiles[2q], qtiles[2q + 1]: the tile_lo and
 * ntiles of query q; *n = the number of such tickets (TRN_ERR_CAPACITY if cap is smaller), ticket t = tickets[3t .. 3t + 2]: the query, the
 * first tile and the end tile (exclusive) it covers, all inside one 2^17-docID run. */
int trn_debug_dense_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid, const trn_query *queries,
                         uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n, char *err, size_t errcap);
/* The same for the flat ANDs with exactly one operand without a resident bitmap (the others with one): their run-major tickets follow the
 * all-bitmap ones (TRN_MIXED_RUNS=0 turns them off).  Same arguments and rows as trn_debug_dense_runs. */
int trn_debug_mixed_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid, const trn_query *queries,
                         uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n, char *err, size_t errcap);
/* The same for the candidate-driven queries (TRN_ROUTE_CANDIDATE): one ticket per 32-block group of the query's lead term, ordered by the
 * 2^17-docID run of the group's first docID, queries ascending within a run; they follow the flat ANDs' run tickets (TRN_CAND_RUNS=0
 * turns them off: the groups then take tickets in query order).  qtiles[2q + 1] = the groups of query q; ticket t = tickets[3t .. 3t + 2]:
 * the query, the group and the group's first docID (the last docID of the block before it plus one; the lead's first docID for group 0). */
int trn_debug_cand_runs(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t max_docid, const trn_query *queries,
                        uint32_t nq, int mode, uint32_t k, uint32_t *qtiles, uint32_t *tickets, uint64_t cap, uint64_t *n, char *err, size_t errcap);

/* Host-only view of the dense-term selection (tests, tooling; no GPU needed): the terms trn_upload_index would keep a resident docID
 * bitmap for on a context that trn_create made with this environment (TRN_DENSE_BITMAPS, TRN_DENSE_BUDGET).  A GOOGLE term qualifies when
 * its bitmap — one bit per docID of its own span, both ends aligned to 2^17 docIDs — is no larger than its chunk; qualifying terms are
 * taken densest first while the bitmaps fit into the budget (default: 25 % of the index bytes).  offsets[0..nterms) receives every term's
 * first 32-bit word in the bitmap array (0xffffffff: none), *nselected the number of terms with a bitmap, *bitmap_bytes their bytes. */
int trn_debug_dense_terms(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t *offsets, uint32_t *nselected,
                          uint64_t *bitmap_bytes, char *err, size_t errcap);

/* The same for the probe bitmaps (TRN_PROBE_BITMAPS, TRN_PROBE_RATIO, TRN_PROBE_BUDGET; TRN_DENSE_BITMAPS=0 turns them off too).  A GOOGLE
 * term without a dense bitmap qualifies when its bitmap is at most TRN_PROBE_RATIO (default 16) times its chunk; qualifying terms are taken
 * densest first (ties: lower term id) while the tier fits into TRN_PROBE_BUDGET x the index bytes (default 2.0) and both tiers together
 * into fewer than 2^32 words.  The tier is laid out behind the dense bitmaps.  offsets[0..nterms) receives the word the candidate-driven
 * conjunction probes each term at: a dense term's dense offset, a probe term's first word, 0xffffffff for a term with neither;
 * *nselected the number of probe terms, *bitmap_bytes their bytes. */
int trn_debug_probe_terms(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, uint32_t *offsets, uint32_t *nselected,
                          uint64_t *bitmap_bytes, char *err, size_t errcap);

/* Debug view (tests, tooling): the resident bitmap of `term` as the upload built it.  *nwords = its 32-bit words (0: the term has none),
 * bit b of word w = docID *base + 32 w + b; the words go to out[0..cap) (TRN_ERR_CAPACITY if cap is smaller). */
int trn_debug_dense_bitmap(trn_ctx *, uint32_t term, uint32_t *out, uint64_t cap, uint64_t *base, uint64_t *nwords);

/* ------------------------------------------------------------------------------------------------ default exec mode
 * == exec_query() with no ExecFlags (exec.h:11-43): MatchedIndexDocumentsFilter::consider(const matched_document &) for every match, with
 * the query terms the match holds and each term's hits (matches.h:34-130).  Which documents match is what DocumentsOnly computes, except
 * that a root Filter over a disjunction really excludes (build_span makes a GenericDocsSetSpan in this mode, exec.cpp:452-505).  The terms
 * of a match follow queryexec_ctx::collect_doc_matching_terms (queryexec_ctx.cpp:382-648): a TERM itself, every child of an AND, the
 * children of an OR / SOME that hold the document, the required side of a NOT, an OPTIONAL's main and its opt where opt holds the document,
 * every term of a PHRASE; duplicates removed; ascending term index.  A query has at most 32 distinct terms and 32 phrase nodes
 * (TRN_ERR_UNSUPPORTED otherwise); a LUCENE source needs its hits.data (trn_upload_hits).  trn_exec_batch refuses this mode. */
#define TRN_MODE_MATCHED_TERMS 4
/* == term_hit (runtime.h:8-11), in its field order */
typedef struct trn_hit {
        uint64_t payload;
        uint16_t pos;
        uint8_t  payload_len;
} trn_hit;
/* Result of trn_exec_matches; pinned buffers owned by the ctx, valid until the next exec call.  Query q owns the matches
 * [doc_offsets[q], doc_offsets[q+1]) of docids (ascending); match m owns the terms [term_offsets[m], term_offsets[m+1]) of terms (the term
 * index, ascending) and freqs; term i owns the hits [hit_offsets[i], hit_offsets[i+1]) of hits. */
typedef struct trn_matches {
        uint32_t        nq;
        uint64_t        total_matches, total_terms, total_hits;
        const uint64_t *doc_offsets;
        const uint32_t *docids;
        const uint64_t *term_offsets;
        const uint32_t *terms;
        const uint32_t *freqs;
        const uint64_t *hit_offsets;
        const trn_hit * hits;
        float           device_ms;  /* CUDA-event time of the whole call: host planning, both passes, the copies and the host synchronisations */
        float           docs_ms;    /* CUDA-event time from the first kernel of the docs pass to the end of its result ordering (no host work) */
        float           count_ms;   /* CUDA-event time of k_collect_count and the scans of terms and hits over the batch (no host work) */
        float           write_ms;   /* CUDA-event time of the k_collect_write launches, summed over the chunks (no copies, no host work) */
        uint32_t        chunks;     /* chunks of matches the write pass ran in (its output buffers are sized per chunk) */
} trn_matches;
/* Per match of the batch the collect pass keeps 28 bytes on the device; the terms and hits are written chunk by chunk of matches
 * (TRN_MATCH_CHUNK, 2^22; halved while a chunk's outputs cannot be allocated) into the pinned result, which is sized once.  As for
 * trn_exec_batch_device, TRN_ERR_CAPACITY means the batch's matches cannot be staged on the device: split the batch.  trn_fetch_results
 * has nothing to fetch after this call (TRN_ERR_STATE). */
int trn_exec_matches(trn_ctx *, const trn_query *queries, uint32_t nq, trn_matches *out);
/* the kernels' hit walker (csrc/hitcursor.h HitWalker) run on the host over one term: for each listed document, whether the term holds it
 * (found[i]) with its freq (counts[i]) and its hits into out[0..cap) (*total = their number) */
int trn_debug_hits(int codec, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hits_bytes, const trn_term *term, const uint32_t *docids, uint32_t n,
                   uint8_t *found, uint32_t *counts, trn_hit *out, uint64_t cap, uint64_t *total, char *err, size_t errcap);

/* Split form used by bench.py / multi-GPU: run on device only, results stay in HBM ... */
int trn_exec_batch_device(trn_ctx *, const trn_query *queries, uint32_t nq, int mode, uint32_t k, trn_result *out_counts_only);
/* ... device pointers of the last SCORED_TOPK run: nq*k u32 docids, nq*k f32 scores (unused slots: docid 0, score -1.0; real scores are >= 0), nq u32 counts */
int trn_last_topk_device(trn_ctx *, void **docids, void **scores, void **counts);

/* ------------------------------------------------------------------------------------------------ per-query document filters
 * == the IndexDocumentsFilter of exec_query (exec.h:50, matches.h:188-201) as docID sets.  A query may name an allow set, a deny set, both
 * or neither; it ignores document d iff
 *         masked(d) || (allow && d not in allow) || (deny && d in deny)
 * which is `documentsFilter->filter(d) || maskedDocumentsRegistry->test(d)` of every exec Handler (exec.cpp:914-932, 1000-1027, 1096-1425).
 * An ignored document is never emitted in any mode, is not counted in match_counts, never takes a top-k candidate slot or moves the
 * threshold, and never reaches trn_exec_matches.  A query with no filter gives the documents and counts it gives without one, also beside
 * filtered queries in one batch; its scores agree to the last-bit spread that k_score_flat's float atomics already have between any two
 * unfiltered runs (so not bit for bit on that route).  Batches without a filtered query run the kernels they ran before.  A query's tiles (and a candidate-driven query's
 * lead-block groups) outside its allow set's first..last docID are not evaluated.
 *
 * One deliberate difference: in the default mode (no ExecFlags) the reference runs a one-term query with a filter through a Handler that
 * sets the term's freq once (exec.cpp:991, 1005-1026), so each match reports freq 1 and hits of a later document, and a document of more
 * than 129 hits overflows its hit buffer.  trn_exec_matches reports the true freq and hits of every match, what the unfiltered run
 * reports for the same document. */

/* A resident docID set (one bit per docID, laid out and padded like the masked-documents bitmap).  Validation follows
 * trn_set_masked_documents: docID 0 is TRN_ERR_ARG, docIDs above max_docid are ignored, order and duplicates do not matter; n == 0 makes
 * the empty set (as an allow set it matches nothing).  Sets live across batches and any number of queries may share one.  A new
 * trn_upload_index invalidates every handle: a stale handle gives TRN_ERR_STATE, a destroyed or unknown one TRN_ERR_ARG.  The handle
 * carries the upload count modulo 65536, so a handle kept across 65536 or more uploads may name a live set of the current index again
 * (never freed memory); callers drop their handles at each upload.
 * TRN_ERR_CAPACITY when the set cannot be allocated (or the context holds TRN_DOCSET_MAX sets, default 65535); the context, its index,
 * its sets and its percolator registry stay usable. */
#define TRN_DOCSET_NONE 0xffffffffu
int trn_docset_create(trn_ctx *, const uint32_t *docids, uint64_t n, uint32_t *handle);
int trn_docset_destroy(trn_ctx *, uint32_t handle);
typedef struct trn_doc_filter {
        uint32_t allow, deny; /* trn_docset_create handles, or TRN_DOCSET_NONE */
} trn_doc_filter;
/* trn_exec_batch / trn_exec_batch_device / trn_exec_matches with filters[0..nq), one per query ({TRN_DOCSET_NONE, TRN_DOCSET_NONE}: no
 * filter).  filters == NULL is the call without them. */
int trn_exec_batch_filtered(trn_ctx *, const trn_query *queries, uint32_t nq, int mode, uint32_t k, const trn_doc_filter *filters, trn_result *out);
int trn_exec_batch_device_filtered(trn_ctx *, const trn_query *queries, uint32_t nq, int mode, uint32_t k, const trn_doc_filter *filters,
                                   trn_result *out_counts_only);
int trn_exec_matches_filtered(trn_ctx *, const trn_query *queries, uint32_t nq, const trn_doc_filter *filters, trn_matches *out);
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
/* trn_encode_google for hits WITH payloads (google_codec.cpp:38-74, the TRACK_PAYLOADS layout): per hit varbyte(delta << 1 | changed),
 * the size byte when it differs from the previous hit's of the same document (0 before a document's first hit), then the payload bytes.
 * The other arguments mean what they mean for trn_encode_google; two more per-hit arrays (HOST pointers, sum(freqs) entries) sit beside
 * positions[]:
 *   payload_lens[]          the payload's size in bytes, 0..8
 *   payloads[]              the payload: the low payload_lens[i] bytes of payloads[i] in memory order (what
 *                           document_proxy::insert(term, pos, {(const uint8_t *)&v, len}) passes)
 * Both NULL: no payloads, the bytes and kernels of trn_encode_google.  A hit at position 0 is written and counted when it has a payload.
 * TRN_ERR_ARG: what trn_encode_google refuses, a position 0 without a payload, a payload of more than 8 bytes, one of the two arrays
 * without the other, or payloads without positions. */
int trn_encode_google_payloads(trn_ctx *, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                               const uint8_t *payload_lens, const uint64_t *payloads, uint32_t block_docs, uint32_t skiplist_step, uint32_t *countdown,
                               uint8_t *out, uint64_t cap, uint64_t *out_bytes, trn_term *terms, float *device_ms);

/* GPU-side Encoder, LUCENE layout == one fresh Codecs::Lucene::IndexSession fed begin_term / begin_document / new_hit / end_document /
 * end_term (lucene_codec.cpp:163-388; FastPFor<4> int-blocks of 128 values, one skiplist entry per full block) for hits without
 * payloads: index and hits.data are BUILT on the device, byte for byte what trn_builder_add_term writes for CODEC_LUCENE (the PFor
 * byte container's padding included: zeros).  term_begin / docids / freqs / positions (HOST pointers) mean what they mean for
 * trn_encode_google; there are no geometry parameters (blocks of 128 documents and of 128 hits, SKIPLIST_STEP = 1 per term).
 *   index_out[index_cap]    the chunks of the terms back to back; *index_bytes their total
 *   hits_out[hits_cap]      hits.data of the terms back to back; *hits_bytes its total (chunk headers hold the offsets into it)
 *   terms[nterms]           the term_index_ctx tuples
 * TRN_ERR_ARG: docID 0 / not ascending, a position 0 / decreasing / >= Limits::MaxPosition (the inputs trn_encode_google refuses).
 * TRN_ERR_CAPACITY: a buffer too small, or an output of 4 GiB or more (u32 offsets); *index_bytes and *hits_bytes are still set.
 * *device_ms (may be NULL): the device time of the kernels and scans, without the host<->device copies. */
int trn_encode_lucene(trn_ctx *, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                      uint8_t *index_out, uint64_t index_cap, uint64_t *index_bytes, uint8_t *hits_out, uint64_t hits_cap, uint64_t *hits_bytes,
                      trn_term *terms, float *device_ms);
/* trn_encode_lucene for hits WITH payloads (lucene_codec.cpp:240-365): a full 128-hit block is intblock(position deltas)
 * intblock(payload sizes) varbyte(sum of the sizes) and the payload bytes; a term's hit tail is varbyte(delta << 1 | changed) [size byte]
 * per hit, `changed` against the previous hit of the tail (0 before its first, across documents), then every payload byte of the tail.
 * payload_lens[] / payloads[] mean what they mean for trn_encode_google_payloads; both NULL: the bytes and kernels of trn_encode_lucene.
 * TRN_ERR_ARG: what trn_encode_lucene refuses, a position 0 without a payload, a payload of more than 8 bytes, one of the two arrays
 * without the other, or payloads without positions.  TRN_ERR_CAPACITY as for trn_encode_lucene. */
int trn_encode_lucene_payloads(trn_ctx *, const uint64_t *term_begin, uint32_t nterms, const uint32_t *docids, const uint32_t *freqs, const uint32_t *positions,
                               const uint8_t *payload_lens, const uint64_t *payloads, uint8_t *index_out, uint64_t index_cap, uint64_t *index_bytes,
                               uint8_t *hits_out, uint64_t hits_cap, uint64_t *hits_bytes, trn_term *terms, float *device_ms);

/* ------------------------------------------------------------------------------------------------ query-token intersections
 * == Trinity::intersect_impl(stopwordsMask, tokens, src, maskedDocumentsRegistry, out) (intersect.h:25-37, intersect.cpp:5-170), one call
 * for a batch of requests over this source, with the context's masked documents as the registry.  Request i has `ngroups` <= 64 groups of
 * synonymous tokens; group g is terms[group_offsets[g] .. group_offsets[g + 1]) (term ids of the uploaded terms table; a term listed twice
 * in one group counts once, as in the reference's unordered_set).  A term that is TRN_EMPTY_TERM or has no documents is unknown: then the
 * query's own mask is not excluded (origMask = 0); with no known token the result is empty.  The result of request i is every
 * {mask, count} of the reference, ordered by popcount descending, count descending, mask ascending (the reference leaves ties in no
 * defined order).  Refusals, never a wrong answer: more than 64 groups or more than 512 known tokens over all groups (a term in two groups
 * counts twice) TRN_ERR_ARG; stopwords_mask != 0 TRN_ERR_UNSUPPORTED (the reference tests it against iterator slots, whose order is
 * not reproducible); more than 65536 distinct masks in a request (TRN_ISECT_MAX_MASKS may lower the limit), or epoch arrays of more
 * than 2^24 entries, TRN_ERR_CAPACITY, naming the request. */
#define TRN_EMPTY_TERM 0xffffffffu
typedef struct trn_isect_req {
        const uint32_t *group_offsets; /* ngroups + 1 */
        const uint32_t *terms;
        uint32_t        ngroups;
        uint64_t        stopwords_mask;
} trn_isect_req;
/* owned by the ctx, valid until the next trn_intersect call: request i owns [offsets[i], offsets[i + 1]) of masks / counts */
typedef struct trn_intersections {
        uint32_t        n;
        uint64_t        total;
        const uint64_t *offsets;
        const uint64_t *masks;
        const uint32_t *counts;
        uint64_t        postings;     /* documents of the known tokens of every request (each token once per group it is in) */
        uint64_t        distinct;     /* distinct masks over the requests (pass A's output) */
        float           masks_ms;     /* CUDA-event time of pass A (k_isect<.., false>), kernel only */
        float           plan_ms;      /* host time of the epoch planner over every request */
        float           count_ms;     /* CUDA-event time of the carries and pass B (k_isect<.., true>), kernels only */
        float           total_ms;     /* host time of the whole call */
} trn_intersections;
int trn_intersect(trn_ctx *, const trn_isect_req *reqs, uint32_t n, trn_intersections *out);
/* Host-only view of the host step between the passes (tests, tooling; no GPU needed): the epochs of one request from its distinct masks and
 * their first docIDs (csrc/isectplan.h).  max_masks = 0: the default limit.  epoch_start[0..*nepochs), epoch_off[0..*nepochs] (entries of
 * epoch e: [epoch_off[e], epoch_off[e + 1]) of snap_mask / snap_slot, cap entries at most), final_mask[0..*nfinal) (n entries suffice for
 * epoch_start and final_mask, n + 1 for epoch_off).  snap_slot: the entry's index in final_mask, -1 when its count is lost. */
int trn_debug_intersect_plan(const uint64_t *masks, const uint32_t *firsts, uint32_t n, uint32_t max_masks, uint32_t *epoch_start, uint32_t *epoch_off,
                             uint64_t *snap_mask, int32_t *snap_slot, uint64_t cap, uint32_t *nepochs, uint64_t *nentries, uint64_t *final_mask, uint32_t *nfinal,
                             char *err, size_t errcap);

/* ------------------------------------------------------------------------------------------------ percolator
 * == Trinity's percolator_query(q).match(proxy) (percolator.h, percolator.cpp) for every registered query and every document of a batch:
 * which stored queries match an incoming document.  A ctx holds at most one registered query set; it needs no uploaded index, and a ctx
 * may hold an index and a registry at once.
 *   Registry   trn_percolator_register: the same trn_qnode trees trn_exec_batch takes; query ids are indices into `queries`; registering
 *              again replaces the set.  Term ids index a percolator vocabulary of `nterms` terms; TRN_EMPTY_TERM is a query term outside it.
 *              term_cost (optional, nterms entries; NULL: all equal), e.g. each term's document frequency, only chooses the anchors.
 *              trn_percolator_add / trn_percolator_remove change the registered set in place (below).
 *   Documents  trn_percolate: document d is tokens[doc_offsets[d] .. doc_offsets[d + 1]) and token i sits at position i + 1; a token
 *              outside the vocabulary is TRN_EMPTY_TERM: it takes up a position and equals no query term, not even TRN_EMPTY_TERM.
 *   Meaning    query q matches document d exactly when percolator_query(q).match(proxy) returns true for the proxy whose match_term(t) says
 *              whether the document holds the token t, and whose match_phrase(t0..tk) whether, at some position p, the tokens at p .. p + k
 *              are t0 .. tk.  TERM / AND / OR / NOT (the first operand and none of the others) / OPTIONAL (its main side) / SOME (at least
 *              `min` >= 1 operands) / PHRASE mean what matchterm / logicaland / logicalor / logicalnot / consttrueexpr beside a conjunction /
 *              matchsome / matchphrase evaluate to.  A const-true expression that does not stand beside a conjunction operand (`<a>`,
 *              `<a> OR <b>`) has no tree form: the front-end drops its wrapper, and the tree means the exec_query meaning.
 *   Refusals   never a wrong answer.  TRN_ERR_ARG, naming the query or document: a malformed tree (the plan compiler's structural checks), a
 *              phrase of more than 16 terms (Limits::MaxPhraseSize), a term id >= nterms other than TRN_EMPTY_TERM, a document token >= nterms
 *              other than TRN_EMPTY_TERM, a document of more than 16383 tokens (positions below Limits::MaxPosition).  TRN_ERR_UNSUPPORTED:
 *              a query whose post-order program needs more than 64 pending operands (an operator with more than 64 operands).
 *              TRN_ERR_STATE: trn_percolate without a registry.  TRN_ERR_CAPACITY: the batch's matches cannot be staged (split the batch).
 *              TRN_PERC_MAX_IDS / TRN_PERC_MAX_ENTRIES lower the id and anchor-entry limits (tests). */
typedef struct trn_percolator_info {
        uint32_t nqueries;
        uint32_t unanchored;     /* queries a match may hold none of the terms of (evaluated for every document) */
        uint32_t never;          /* queries no document can match (never evaluated) */
        uint32_t next_id;        /* the id the next added query gets (nqueries right after a registration) */
        uint64_t anchor_entries; /* (term, query) entries of the term -> anchored-queries index */
        uint64_t device_bytes;   /* the registry in HBM: the bytes uploaded after a registration, the buffers' capacity after an add or remove */
} trn_percolator_info;
/* nqueries / unanchored / never / anchor_entries describe the live queries (issued and not removed). */
int trn_percolator_register(trn_ctx *, const trn_query *queries, uint32_t nq, uint32_t nterms, const uint32_t *term_cost, trn_percolator_info *out);
/* In-place changes of the registered set.  After any sequence of register / add / remove, trn_percolate returns exactly what registering
 * the live queries fresh returns, with ids mapped through the live ids: the same matches per document, ascending id, and the same
 * `candidates`.  The anchor index and the unanchored list are rebuilt on the device into what a fresh registration of every issued query
 * would hold minus the removed ones; k_perc reads them as it reads a registration's.
 *   trn_percolator_add     appends nq queries with the ids *first_id .. *first_id + nq - 1 (ids are never reused until the next
 *                          trn_percolator_register, which starts again at 0).  Same trees, vocabulary (nterms) and term_cost as the
 *                          registration: growing the vocabulary or changing the costs means registering again.
 *   trn_percolator_remove  removes live queries: no later trn_percolate returns them.
 * Refusals, atomic: a refused call leaves the registry, and the last trn_percolate result, exactly as they were.  trn_percolator_add returns
 * the codes trn_percolator_register returns for the same input, naming the query by its index in the batch; TRN_ERR_CAPACITY when ids
 * would reach 0xFFFFFFFF (it pads the sort in k_perc, so it is never an id) or anchor entries 2^32.  trn_percolator_remove: TRN_ERR_ARG,
 * naming the id, for an id never issued, already removed or given twice.  Either: TRN_ERR_STATE without a registry; TRN_ERR_CAPACITY /
 * TRN_ERR_CUDA when device memory cannot be allocated (the new index is built in new buffers and replaces the old one only on success).
 * nq == 0 / n == 0: a no-op.
 * Memory: the programs of added queries are appended (a full buffer is replaced by one twice its size); when the program words of removed
 * queries outnumber the live ones, the program storage is compacted on the device.  The per-id query table (16 B per id ever issued) and
 * the bitmap width of a document with more than 4096 matches (next_id / 32 words) grow with next_id until the next registration. */
int trn_percolator_add(trn_ctx *, const trn_query *queries, uint32_t nq, uint32_t *first_id, trn_percolator_info *out);
int trn_percolator_remove(trn_ctx *, const uint32_t *ids, uint32_t n, trn_percolator_info *out);
/* CUDA-event time of the device work of the last successful trn_percolator_add / trn_percolator_remove (its uploads, program copies and
 * rebuild kernels) and its host time, ms. */
int trn_percolator_last_update(trn_ctx *, float *device_ms, float *host_ms);
/* Debug view (tests, tooling): copies the resident index and unanchored list to the host.  csr_off: *nterms + 1 entries; csr: 2 words per
 * entry (query id, anchor ordinal), entry e of term t at csr_off[t] <= e < csr_off[t + 1]; unanchored: ascending ids.  Any output may be
 * NULL (then *nterms, *nentries and *nunanchored still report the sizes); cap / ucap entries at most, TRN_ERR_CAPACITY beyond. */
int trn_debug_percolator_registry(trn_ctx *, uint32_t *csr_off, uint32_t *csr, uint64_t cap, uint32_t *unanchored, uint64_t ucap, uint32_t *nterms,
                                  uint64_t *nentries, uint64_t *nunanchored);
/* owned by the ctx, valid until the next trn_percolate: document d owns [offsets[d], offsets[d + 1]) of queries (ascending, no duplicates) */
typedef struct trn_percolation {
        uint32_t        ndocs;
        uint32_t        long_docs;  /* documents of more than 512 tokens (the long launch: larger shared tables) */
        uint32_t        dense_docs; /* documents of more than 4096 matches (ids emitted from a bitmap over the query ids, not sorted in shared memory) */
        uint32_t        pad;
        uint64_t        total;
        const uint64_t *offsets;
        const uint32_t *queries;
        uint64_t        candidates; /* (document, query) pairs evaluated */
        float           count_ms;   /* CUDA-event time of the count pass and the scan of the counts (kernels only) */
        float           write_ms;   /* CUDA-event time of the write pass (kernels only) */
        float           total_ms;   /* host time of the whole call */
} trn_percolation;
int trn_percolate(trn_ctx *, const uint64_t *doc_offsets, const uint32_t *tokens, uint32_t ndocs, trn_percolation *out);
/* Host-only view of the registration planner (csrc/percplan.h; tests, tooling; no GPU needed): status[q] = 0 anchored, 1 unanchored, 2 no
 * document can match; query q's anchor cover (ascending term id) = cover_terms[cover_off[q] .. cover_off[q + 1]) (nq + 1 offsets, at most cap
 * terms: TRN_ERR_CAPACITY beyond, *ncover = the number needed).  The refusals of trn_percolator_register. */
int trn_debug_percolator_plan(const trn_query *queries, uint32_t nq, uint32_t nterms, const uint32_t *term_cost, uint8_t *status, uint32_t *cover_off,
                              uint32_t *cover_terms, uint64_t cap, uint64_t *ncover, char *err, size_t errcap);

/* ------------------------------------------------------------------------------------------------ indexer
 * == SegmentIndexSession begin / insert / commit (indexer.h, indexer.cpp:14-153, 311-564) for one batch of tokenised documents: the
 * documents are inverted on the device (a keys-only radix sort), encoded by the device encoders and come back as the `index` (and LUCENE
 * `hits.data`) bytes the reference's commit() would have written for the same documents; trn_segment_write makes a segment directory of them.
 *   docids[ndocs]            the documents' ids, in any order, > 0, no id twice
 *   doc_offsets[ndocs + 1]   document d is tokens[doc_offsets[d] .. doc_offsets[d + 1]); doc_offsets[0] = 0; an empty document is legal and
 *                            is not counted in docs_cnt (indexer.cpp:361-364)
 *   tokens[]                 term ids below nterms; term t stands for the reference's transient term id t + 1, which fixes the order of the
 *                            chunks in the index: by (t + 1) & 31, then by t (indexer.cpp:388, 402-410, 423)
 *   positions[]              the position of every token, in any order inside a document, equal positions allowed; NULL: token i of a
 *                            document sits at position i + 1 (trn_percolate's convention)
 * All pointers are HOST pointers.  The GOOGLE geometry is the reference's (32 / 8, a fresh countdown).  The hits carry no payloads.
 * Refusals, never a wrong answer, each naming the document or term.  TRN_ERR_ARG: docID 0, a docID twice, a token >= nterms, doc_offsets
 * not ascending, a position >= 16384 (Limits::MaxPosition), more than 65535 hits of one term in one document or more than 65535 distinct
 * terms in one document (uint16_t counts of the reference), nterms > 2^24, ndocs > 2^26.  TRN_ERR_UNSUPPORTED: a position 0 (a hit without
 * a position).  TRN_ERR_CAPACITY: an index or hits.data of 4 GiB or more, or working memory that cannot be allocated (split the batch).
 * A refused call leaves the context's uploaded index, percolator registry and earlier results as they were. */
typedef struct trn_indexed { /* owned by the ctx, valid until the next trn_index_documents */
        const uint8_t * index;
        uint64_t        index_bytes;
        const uint8_t * hits; /* LUCENE hits.data; 0 bytes for GOOGLE */
        uint64_t        hits_bytes;
        const trn_term *terms; /* by term id; documents == 0: the term has no posting and is not in the segment */
        uint32_t        nterms;
        uint32_t        docs_cnt, total_terms; /* IndexSource::field_statistics (indexer.cpp:366, 446, 465, 473) */
        uint64_t        sum_terms_docs, sum_term_hits;
        uint32_t        max_docid;
        uint32_t        sort_passes; /* radix passes run (documents + tokens): one per group of up to 8 key bits that can be non-zero */
        float           sort_ms, postings_ms, encode_ms; /* CUDA events of the kernels alone: ranks + keys + sort, the postings pass, the encoder */
        float           total_ms;                        /* host time of the whole call, copies included */
} trn_indexed;
int trn_index_documents(trn_ctx *, int codec, const uint32_t *docids, const uint64_t *doc_offsets, const uint32_t *tokens, const uint32_t *positions,
                        uint32_t ndocs, uint32_t nterms, trn_indexed *out);
/* trn_index_documents for hits WITH payloads (document_proxy::insert(term, pos, payload), indexer.h:115-147; indexer.cpp:14-30): two more
 * per-token arrays (HOST pointers) beside tokens[] / positions[]:
 *   payload_lens[]           the token's payload size in bytes, 0..8
 *   payloads[]               its payload: the low payload_lens[i] bytes of payloads[i] in memory order
 * Both NULL: trn_index_documents.  The device encoders write the hits with their payloads (trn_encode_google_payloads /
 * trn_encode_lucene_payloads).  The refusals of trn_index_documents, except that a position 0 WITH a payload is indexed (the reference's
 * encoders write it, and it counts in the freq and sum_term_hits), and:
 *   TRN_ERR_ARG          a payload of more than 8 bytes (indexer.cpp:26), one of the two arrays without the other
 *   TRN_ERR_UNSUPPORTED  two tokens of one document with the same term and position and different payloads, naming the document and term
 *                        (the reference orders them with an unstable sort, indexer.cpp:55-57; equal payloads are fine); a position 0
 *                        without a payload
 *   TRN_ERR_CAPACITY     more than 2^32 - 1 tokens in the call (split the batch) */
int trn_index_documents_payloads(trn_ctx *, int codec, const uint32_t *docids, const uint64_t *doc_offsets, const uint32_t *tokens, const uint32_t *positions,
                                 const uint8_t *payload_lens, const uint64_t *payloads, uint32_t ndocs, uint32_t nterms, trn_indexed *out);
/* Host code, no device: writes the segment directory `dir` as persist_segment / persist_terms do (indexer.cpp:241-300, codecs.cpp:17-27,
 * terms.cpp:126-172 pack_terms, docidupdates.cpp:8-73 pack_updates): `index`, `hits.data` (LUCENE), `terms.data`, `terms.idx`, `id`, and
 * `updated_documents.ids` when nupdated > 0.  terms[i] <-> names[i]; terms with documents == 0 are left out.  updated_docids = the ids of
 * the documents this segment replaces in older segments plus the erased ids.  The last component of `dir` must be a number, the segment's
 * generation (segment_index_source.cpp:18-21); the directory is created when missing.  TRN_ERR_ARG: such a name, an empty name or one
 * longer than 64 bytes (Limits::MaxTermLength), two equal names, an id twice in updated_docids (the reference's "Already committed
 * document").  TRN_ERR_STATE: a file cannot be written. */
int trn_segment_write(const char *dir, int codec, const uint8_t *index, uint64_t index_bytes, const uint8_t *hits, uint64_t hits_bytes, const trn_term *terms,
                      const char *const *names, uint32_t nterms, uint64_t sum_term_hits, uint32_t total_terms, uint64_t sum_terms_docs, uint32_t docs_cnt,
                      const uint32_t *updated_docids, uint64_t nupdated, char *err, size_t errcap);

/* ------------------------------------------------------------------------------------------------ merge
 * == MergeCandidatesCollection commit() + merge() (merge.cpp:6-35, 40-416) into a fresh IndexSession of out_codec: N index sources
 * (generations) fold into one segment.  Candidates run newest generation first; candidate i's masked documents are the union of the
 * updated_docids of every NEWER candidate.  Output terms come in terms_cmp order (bytewise, a prefix first); per term:
 *   skip      one holder with 0 documents;
 *   append    one holder of out_codec with an empty registry, disable_optimizations == 0: its chunk copied (LUCENE: with its positions
 *             chunk, the header's hitsDataOffset rewritten);
 *   re-encode every other case: of every docID, the newest holder's posting is written unless that holder's registry masks it; older
 *             holders of the docID are never written.  A re-encoded term left without postings still writes its header (GOOGLE 2 bytes,
 *             LUCENE 14) and is not an output term.
 * Per source: names in terms_cmp order (strictly ascending, 1..64 bytes), terms[i] <-> names[i], LUCENE sources with their hits.data.
 * All pointers are HOST pointers.  The re-encode path runs on the device: decode with hits, keep / rank, scatter, the device encoders,
 * one assembly copy.  Refusals, never a wrong answer, each naming the source (and term): TRN_ERR_ARG more than 128 sources, two equal
 * generations, a bad name or order, a tuple outside its source's bytes, a LUCENE source without hits.data, a malformed chunk;
 * TRN_ERR_UNSUPPORTED a hit with a payload, or at a position outside 1..16383, of a posting that is written re-encoded (appended chunks
 * keep their payloads; postings not written are never read); TRN_ERR_CAPACITY an output of 4 GiB or more, or
 * working memory that cannot be allocated.  n = 0: an empty result.  A refused call leaves the context as it was.
 * trn_merge_sources_payloads: the same call, arguments, result and refusals, except that a re-encoded posting's hits are written with
 * their payloads (new_hit(pos, {payload, len}), merge.cpp:221-232, 352-361: the low len bytes of the payload) and a hit at position 0
 * WITH a payload is written and counts in sum_term_hits, as trn_index_documents_payloads writes it.  Its refusals of a written re-encoded
 * posting: TRN_ERR_UNSUPPORTED a hit at position 0 without a payload, or above 16383; TRN_ERR_FORMAT a stored payload length above 8
 * (a malformed source).  A merge none of whose written re-encoded hits carries a payload writes what trn_merge_sources writes. */
#define TRN_MERGE_MAX_SOURCES 128
typedef struct trn_merge_source {
        int                codec;
        uint64_t           generation;
        const uint8_t *    index;
        uint64_t           index_bytes;
        const uint8_t *    hits; /* LUCENE hits.data */
        uint64_t           hits_bytes;
        const trn_term *   terms;
        const char *const *names;
        uint32_t           nterms;
        const uint32_t *   updated_docids; /* replaced and erased documents of this generation, any order */
        uint64_t           nupdated;
} trn_merge_source;
typedef struct trn_merged { /* owned by the ctx, valid until the next trn_merge_sources(_payloads) */
        const uint8_t * index;
        uint64_t        index_bytes;
        const uint8_t * hits; /* LUCENE hits.data */
        uint64_t        hits_bytes;
        const trn_term *terms;       /* output terms in output (terms_cmp) order */
        const uint32_t *term_source; /* the source (index into src[]) and that source's term index whose name term i carries */
        const uint32_t *term_index;
        uint32_t        nterms;
        uint32_t        total_terms, docs_cnt; /* docs_cnt: distinct docIDs holding an output posting (merge() leaves it to the caller) */
        uint64_t        sum_terms_docs, sum_term_hits; /* only the postings of the two decode loops count (merge.cpp:224-225, 363-364) */
        uint32_t        appended, reencoded, orphaned;
        uint64_t        postings_read, postings_written;
        float           decode_ms, merge_ms, encode_ms, assemble_ms; /* CUDA events of the phases' kernels */
        float           total_ms;                                    /* host time of the whole call, copies included */
} trn_merged;
int trn_merge_sources(trn_ctx *, int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, trn_merged *out);
int trn_merge_sources_payloads(trn_ctx *, int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, trn_merged *out);
/* Host-only view of the merge planner (csrc/mergeplan.h; no GPU).  Arrays sized by the caller: order[n] = source of candidate i (newest
 * first); per output term k (at most Σ nterms): route[k] (0 append, 1 re-encode), stats[k] (1: its postings count toward sum_terms_docs /
 * sum_term_hits), parts [part_off[k], part_off[k + 1]) (nout + 1 offsets) of part_cand / part_term (candidate, term of that candidate's
 * source; newest first); the registries as the sorted distinct updated docIDs upd_docid[nupd] (at most Σ nupdated) with upd_first[i] =
 * the newest candidate that updates it: candidate j masks d iff upd_first(d) < j.  countdown_phase: the GOOGLE skiplist phase the
 * re-encoded terms start from.  The refusals of trn_merge_sources that need no postings. */
int trn_debug_merge_plan(int out_codec, const trn_merge_source *src, uint32_t n, int disable_optimizations, uint32_t *order, uint8_t *route,
                         uint8_t *stats, uint32_t *part_off, uint32_t *part_cand, uint32_t *part_term, uint32_t *nout, uint64_t *nparts, uint32_t *upd_docid,
                         uint32_t *upd_first, uint64_t *nupd, uint32_t *countdown_phase, char *err, size_t errcap);

#ifdef __cplusplus
}
#endif
#endif
