// Host-side half of the C ABI: index builder, synthetic workload generator, query front-end, BM25 weights.
// (The device half lives in engine.cu.)  No reference code is linked here; formats are pinned by tests against oracle/_ref.
#include "../../include/trinity_b200.h"
#include "chunkplan.h"
#include "codecs.h"
#include "dirlookup.h"
#include "hitcursor.h"
#include "varbyte.h"
#include <algorithm>
#include <atomic>
#include <cctype>
#include <cmath>
#include <cstring>
#include <memory>
#include <stdexcept>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

using namespace trn;

static constexpr uint32_t kEmptyTerm = 0xffffffffu; // == device_types.h
static constexpr int      kConstTrue = 100;        // parser-internal node kind for <expr>

// =================================================================================================== builder
struct trn_builder {
        Codecs::IndexSession             sess;
        std::unique_ptr<Codecs::Encoder> enc;
        std::string                      err;
        explicit trn_builder(Codec c)
            : sess{c}, enc{Codecs::new_encoder(&sess)} {
        }
};

template <class F> static int guarded(trn_builder *b, F &&f) {
        if (!b)
                return TRN_ERR_ARG;
        try {
                f();
                return TRN_OK;
        } catch (const std::exception &e) {
                b->err = e.what();
        } catch (...) {
                b->err = "unknown error";
        }
        return TRN_ERR_ARG;
}

extern "C" int trn_builder_create(int codec, trn_builder **out) {
        if (!out || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        *out = new trn_builder(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene);
        return TRN_OK;
}
extern "C" void trn_builder_destroy(trn_builder *b) {
        delete b;
}
extern "C" const char *trn_builder_last_error(trn_builder *b) {
        return b ? b->err.c_str() : "null builder";
}
extern "C" int trn_builder_begin_term(trn_builder *b) {
        return guarded(b, [&] { b->enc->begin_term(); });
}
extern "C" int trn_builder_begin_document(trn_builder *b, uint32_t docid) {
        return guarded(b, [&] { b->enc->begin_document(docid); });
}
extern "C" int trn_builder_new_hit(trn_builder *b, uint32_t position, const uint8_t *payload, uint8_t payload_len) {
        return guarded(b, [&] { b->enc->new_hit(position, payload, payload_len); });
}
extern "C" int trn_builder_end_document(trn_builder *b) {
        return guarded(b, [&] { b->enc->end_document(); });
}
extern "C" int trn_builder_end_term(trn_builder *b, trn_term *out) {
        return guarded(b, [&] {
                term_index_ctx t;
                b->enc->end_term(&t);
                if (out) {
                        out->documents = t.documents;
                        out->chunk_off = t.offset;
                        out->chunk_len = t.size;
                }
        });
}
extern "C" int trn_builder_add_term(trn_builder *b, const uint32_t *docids, const uint32_t *freqs, uint32_t n, const uint32_t *positions, trn_term *out) {
        return guarded(b, [&] {
                size_t pi{0};
                b->enc->begin_term();
                for (uint32_t i = 0; i < n; ++i) {
                        b->enc->begin_document(docids[i]);
                        for (uint32_t k = 0; k < freqs[i]; ++k)
                                b->enc->new_hit(positions ? positions[pi++] : k + 1);
                        b->enc->end_document();
                }
                term_index_ctx t;
                b->enc->end_term(&t);
                if (out) {
                        out->documents = t.documents;
                        out->chunk_off = t.offset;
                        out->chunk_len = t.size;
                }
        });
}
extern "C" int trn_builder_set_google_skiplist_countdown(trn_builder *b, uint32_t countdown) {
        return guarded(b, [&] {
                if (b->sess.codec != Codec::Google || countdown == 0 || countdown > Codecs::Google::SKIPLIST_STEP)
                        throw std::invalid_argument("countdown only applies to the GOOGLE codec, range 1..8");
                static_cast<Codecs::Google::Encoder *>(b->enc.get())->skiplistEntryCountdown = countdown;
        });
}
extern "C" int trn_builder_set_google_block(trn_builder *b, uint32_t block_docs, uint32_t skiplist_step) {
        return guarded(b, [&] {
                if (b->sess.codec != Codec::Google || block_docs == 0 || block_docs > Codecs::Google::MAX_N || skiplist_step == 0)
                        throw std::invalid_argument("google block size must be in 1..128 and the skiplist step >= 1 (GOOGLE codec only)");
                auto *e = static_cast<Codecs::Google::Encoder *>(b->enc.get());
                e->blockDocs = block_docs;
                e->skiplistStep = e->skiplistEntryCountdown = skiplist_step;
        });
}
extern "C" int trn_builder_index(trn_builder *b, const uint8_t **index, uint64_t *nbytes) {
        if (!b || !index || !nbytes)
                return TRN_ERR_ARG;
        *index  = b->sess.indexOut.data();
        *nbytes = b->sess.indexOut.size();
        return TRN_OK;
}
extern "C" int trn_builder_hits(trn_builder *b, const uint8_t **hits, uint64_t *nbytes) {
        if (!b || !hits || !nbytes)
                return TRN_ERR_ARG;
        *hits   = b->sess.positionsOut.data();
        *nbytes = b->sess.positionsOut.size();
        return TRN_OK;
}

extern "C" int trn_directory_probe(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *term, uint32_t *blk_last, uint32_t *blk_off, uint32_t cap,
                                   uint32_t *nblocks, uint32_t *first_doc, char *err, size_t errcap) {
        if (!index || !term || !nblocks || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        try {
                term_index_ctx t;
                t.documents = term->documents;
                t.offset    = term->chunk_off;
                t.size      = term->chunk_len;
                BlockDirectory d;
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, &t, 1, 1, d);
                *nblocks = d.terms[0].nblocks;
                if (first_doc)
                        *first_doc = d.terms[0].first_doc;
                for (uint32_t i = 0; i < d.blk_last.size() && i < cap; ++i) {
                        if (blk_last)
                                blk_last[i] = d.blk_last[i];
                        if (blk_off)
                                blk_off[i] = d.blk_off[i];
                }
                return TRN_OK;
        } catch (const std::exception &e) {
                if (err && errcap) {
                        std::strncpy(err, e.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_FORMAT;
        }
}

extern "C" int trn_directory_lookup(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *term, const uint32_t *docids, uint32_t n, uint32_t *blocks,
                                    uint32_t *tf_shift, uint32_t *tf_entries, char *err, size_t errcap) {
        if (!index || !term || (n && (!docids || !blocks)) || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        try {
                term_index_ctx t;
                t.documents = term->documents;
                t.offset    = term->chunk_off;
                t.size      = term->chunk_len;
                BlockDirectory d;
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, &t, 1, 1, d);
                const auto &T = d.terms[0];
                if (tf_shift)
                        *tf_shift = T.tf_shift;
                if (tf_entries)
                        *tf_entries = uint32_t(d.tile_first.size());
                for (uint32_t i = 0; i < n; ++i)
                        blocks[i] = T.nblocks ? dir_first_block_ge(d.blk_last.data() + T.dir_begin, d.tile_first.data() + T.tf_begin, T.nblocks, T.first_doc, T.last_doc,
                                                                   T.tf_base, T.tf_shift, docids[i])
                                              : 0u;
                return TRN_OK;
        } catch (const std::exception &e) {
                if (err && errcap) {
                        std::strncpy(err, e.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_FORMAT;
        }
}

// The kernels' own position cursors (csrc/hitcursor.h) run on the host: the positions of every listed document of one term, through the
// load-time directories — what phrase.cuh reads per (candidate, term).  positions[] receives them document after document; counts[i] =
// how many document i holds (0: the term does not hold it).
extern "C" int trn_debug_positions(int codec, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hbytes, const trn_term *term, const uint32_t *docids,
                                   uint32_t n, uint32_t *counts, uint32_t *positions, uint64_t cap, uint64_t *total, char *err, size_t errcap) {
        if (!index || !term || !total || (n && (!docids || !counts)) || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        try {
                term_index_ctx t;
                t.documents = term->documents;
                t.offset    = term->chunk_off;
                t.size      = term->chunk_len;
                BlockDirectory d;
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, &t, 1, 1, d);
                HitsDirectory hd;
                HitTerm       ht{0, 0};
                if (codec == TRN_CODEC_LUCENE) {
                        build_hits_directory(index, nbytes, hits, hbytes, &t, 1, d, 1, hd);
                        ht = HitTerm{hd.hb_begin[0], hd.sum_hits[0]};
                }
                HitsView v;
                v.index      = index;
                v.blk_last   = d.blk_last.data();
                v.blk_off    = d.blk_off.data();
                v.tile_first = d.tile_first.data();
                v.hits       = hits;
                v.hit_base   = hd.hit_base.data();
                v.hblk_off   = hd.hblk_off.data();
                v.hit_term   = &ht;
                v.codec      = codec == TRN_CODEC_GOOGLE ? 0 : 1;
                const auto &T = d.terms[0];
                PhraseTerm  pt;
                pt.dir    = T.dir_begin;
                pt.nb     = T.nblocks;
                pt.docs   = T.documents;
                pt.first  = T.first_doc;
                pt.last   = T.last_doc;
                pt.tfb    = T.tf_begin;
                pt.tfbase = T.tf_base;
                pt.tfs    = T.tf_shift;
                pt.id     = 0;
                uint64_t k{0};
                for (uint32_t i = 0; i < n; ++i) {
                        HitCursor c = hit_cursor(v, pt, docids[i]);
                        counts[i]   = c.left;
                        while (c.left) {
                                const uint32_t pos = c.next();
                                if (k < cap)
                                        positions[k] = pos;
                                ++k;
                        }
                }
                *total = k;
                return k > cap ? TRN_ERR_CAPACITY : TRN_OK;
        } catch (const std::exception &e) {
                if (err && errcap) {
                        std::strncpy(err, e.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_FORMAT;
        }
}

extern "C" int trn_debug_hits(int codec, const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hbytes, const trn_term *term, const uint32_t *docids,
                              uint32_t n, uint8_t *found, uint32_t *counts, trn_hit *out, uint64_t cap, uint64_t *total, char *err, size_t errcap) {
        if (!index || !term || !total || (n && (!docids || !counts || !found)) || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        try {
                term_index_ctx t;
                t.documents = term->documents;
                t.offset    = term->chunk_off;
                t.size      = term->chunk_len;
                BlockDirectory d;
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, &t, 1, 1, d);
                HitsDirectory hd;
                HitTerm       ht{0, 0};
                if (codec == TRN_CODEC_LUCENE) {
                        build_hits_directory(index, nbytes, hits, hbytes, &t, 1, d, 1, hd);
                        ht = HitTerm{hd.hb_begin[0], hd.sum_hits[0]};
                }
                HitsView v;
                v.index      = index;
                v.blk_last   = d.blk_last.data();
                v.blk_off    = d.blk_off.data();
                v.tile_first = d.tile_first.data();
                v.hits       = hits;
                v.hit_base   = hd.hit_base.data();
                v.hblk_off   = hd.hblk_off.data();
                v.hit_term   = &ht;
                v.codec      = codec == TRN_CODEC_GOOGLE ? 0 : 1;
                const auto &T = d.terms[0];
                PhraseTerm  pt;
                pt.dir    = T.dir_begin;
                pt.nb     = T.nblocks;
                pt.docs   = T.documents;
                pt.first  = T.first_doc;
                pt.last   = T.last_doc;
                pt.tfb    = T.tf_begin;
                pt.tfbase = T.tf_base;
                pt.tfs    = T.tf_shift;
                pt.id     = 0;
                uint64_t k{0};
                for (uint32_t i = 0; i < n; ++i) {
                        uint32_t freq{0};
                        found[i]  = term_holds(v, pt, docids[i], freq) ? 1 : 0;
                        counts[i] = freq;
                        if (!found[i] || !freq)
                                continue;
                        HitWalker w;
                        w.init(v, pt, docids[i]);
                        while (w.c.left) {
                                uint32_t       len{0};
                                const uint32_t pos = w.next(len);
                                if (k < cap && out)
                                        out[k] = trn_hit{w.payload, uint16_t(pos), uint8_t(len)};
                                ++k;
                        }
                }
                *total = k;
                return k > cap ? TRN_ERR_CAPACITY : TRN_OK;
        } catch (const std::exception &e) {
                if (err && errcap) {
                        std::strncpy(err, e.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_FORMAT;
        }
}

extern "C" int trn_directory_stats(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, int threads, uint64_t *directory_bytes,
                                   uint64_t *total_blocks, uint64_t *table_entries, char *err, size_t errcap) {
        if (!index || !terms || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE))
                return TRN_ERR_ARG;
        try {
                std::vector<term_index_ctx> t(nterms);
                for (uint32_t i = 0; i < nterms; ++i) {
                        t[i].documents = terms[i].documents;
                        t[i].offset    = terms[i].chunk_off;
                        t[i].size      = terms[i].chunk_len;
                }
                BlockDirectory d;
                build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, t.data(), nterms, std::max(1, threads), d);
                uint64_t blocks{0};
                for (const auto &x : d.terms)
                        blocks += x.nblocks;
                if (directory_bytes)
                        *directory_bytes = d.bytes();
                if (total_blocks)
                        *total_blocks = blocks;
                if (table_entries)
                        *table_entries = d.tile_first.size();
                return TRN_OK;
        } catch (const std::exception &e) {
                if (err && errcap) {
                        std::strncpy(err, e.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_FORMAT;
        }
}

// =================================================================================================== synthetic index
namespace {
inline uint64_t splitmix64(uint64_t &s) {
        uint64_t z = (s += 0x9E3779B97F4A7C15ull);
        z          = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
        z          = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
        return z ^ (z >> 31);
}

inline uint32_t synth_df(uint32_t ndocs, uint32_t rank, uint32_t min_df) {
        const uint64_t z = uint64_t(ndocs) / (2ull * rank); // floor(0.5 * N / r)
        return uint32_t(std::min<uint64_t>(ndocs, std::max<uint64_t>(min_df, z)));
}

// Calls f(docid, freq, stateForPositions) for each posting of term `rank`
template <class F> void synth_term(uint32_t ndocs, uint32_t rank, uint32_t min_df, uint64_t seed, F &&f) {
        const uint32_t df = synth_df(ndocs, rank, min_df);
        uint64_t       s  = seed ^ uint64_t(rank);
        uint64_t       s2 = (seed ^ uint64_t(rank)) * 0xD1342543DE82EF95ull + 0x2545F4914F6CDD1Dull;
        const double   p  = double(df) / double(ndocs);
        const double   il = p < 1.0 ? 1.0 / std::log1p(-p) : 0.0;
        uint64_t       doc{0};
        for (uint32_t i = 0; i < df; ++i) {
                const uint64_t x = splitmix64(s);
                uint64_t       gap{1};
                if (p < 1.0) {
                        const double u = double((x >> 11) + 1) * (1.0 / 9007199254740992.0); // (0, 1]
                        const double g = std::floor(std::log(u) * il);
                        gap            = 1 + uint64_t(std::min(g, 4.0e9));
                }
                const uint64_t maxdoc = uint64_t(ndocs) - (df - 1 - i);
                doc                   = std::min(doc + gap, maxdoc);
                const uint32_t geo    = uint32_t(__builtin_ctzll((x & 0x7ffull) | 0x800ull));
                const uint32_t freq   = 1 + std::min<uint32_t>(7, geo);
                f(uint32_t(doc), freq, splitmix64(s2));
        }
}

// positions of one document: cumulative steps 2..17 (== 1 + u(1..16)), < Limits::MaxPosition (trinity_limits.h:15)
inline uint32_t synth_pos_step(uint64_t y, uint32_t h) {
        return 2u + uint32_t((y >> (4u * h)) & 15u);
}
} // namespace

struct trn_synth {
        Codec                 codec;
        std::vector<uint8_t>  index, hits;
        std::vector<trn_term> terms;
        uint64_t              sumHits{0};
};

extern "C" int trn_synth_build(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, trn_synth **out) {
        return trn_synth_build_shard(codec, ndocs, nterms, min_df, seed, with_hits, threads, 1, ndocs, out);
}

// docID-range shard [doc_lo, doc_hi] of the same index: every term keeps only its postings inside the range (== one IndexSource of
// an IndexSourcesCollection partitioned by docID, index_source.h:191-238; SURVEY.md 8e).  docIDs stay global.
extern "C" int trn_synth_build_shard(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, uint32_t doc_lo,
                                     uint32_t doc_hi, trn_synth **out) {
        return trn_synth_build_ex(codec, ndocs, nterms, min_df, seed, with_hits, threads, doc_lo, doc_hi, Codecs::Google::N, Codecs::Google::SKIPLIST_STEP, out);
}

// the same with the two compile-time constants of the GOOGLE format (google_codec.h:17-20: N, SKIPLIST_STEP) as parameters: the decode
// sweep of BASELINE.json configs[4] (other values are not the reference's on-disk format; the exec kernels refuse such an index)
extern "C" int trn_synth_build_ex(int codec, uint32_t ndocs, uint32_t nterms, uint32_t min_df, uint64_t seed, int with_hits, int threads, uint32_t doc_lo,
                                  uint32_t doc_hi, uint32_t google_block_docs, uint32_t google_skiplist_step, trn_synth **out) {
        if (!out || !ndocs || !nterms || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || doc_lo == 0 || doc_lo > doc_hi || google_block_docs == 0 ||
            google_block_docs > Codecs::Google::MAX_N || google_skiplist_step == 0)
                return TRN_ERR_ARG;
        const uint32_t GN = google_block_docs, GS = google_skiplist_step;
        const Codec cd = codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene;
        const bool  whole = doc_lo <= 1 && doc_hi >= ndocs;
        if (threads < 1)
                threads = int(std::max(1u, std::thread::hardware_concurrency()));
        // documents of every term inside the range (analytic for the whole index, counted by a generation-only pass otherwise)
        std::vector<uint32_t> dfIn(nterms);
        if (whole) {
                for (uint32_t r = 1; r <= nterms; ++r)
                        dfIn[r - 1] = synth_df(ndocs, r, min_df);
        } else {
                std::atomic<uint32_t> nx{0};
                auto                  counter = [&] {
                        for (;;) {
                                const uint32_t i = nx.fetch_add(1);
                                if (i >= nterms)
                                        break;
                                uint32_t c{0};
                                synth_term(ndocs, i + 1, min_df, seed, [&](uint32_t doc, uint32_t, uint64_t) { c += doc >= doc_lo && doc <= doc_hi; });
                                dfIn[i] = c;
                        }
                };
                std::vector<std::thread> ths;
                for (int i = 1; i < threads; ++i)
                        ths.emplace_back(counter);
                counter();
                for (auto &t : ths)
                        t.join();
        }
        struct Part {
                std::vector<uint8_t> index, hits;
                term_index_ctx       t;
                uint64_t             hitsCnt{0};
        };
        std::vector<Part> parts(nterms);
        // Google: the skiplist countdown carries over between terms (google_codec.h:57): phase = committed blocks so far mod 8
        std::vector<uint32_t> countdown(nterms, GS);
        {
                uint64_t blocks{0};
                for (uint32_t r = 1; r <= nterms; ++r) {
                        countdown[r - 1] = GS - uint32_t(blocks % GS);
                        blocks += (dfIn[r - 1] + GN - 1) / GN;
                }
        }
        std::atomic<uint32_t> next{0};
        std::atomic<bool>     failed{false};
        auto                  worker = [&] {
                for (;;) {
                        const uint32_t i = next.fetch_add(1);
                        if (i >= nterms || failed.load())
                                break;
                        try {
                                Codecs::IndexSession             sess(cd);
                                std::unique_ptr<Codecs::Encoder> enc(Codecs::new_encoder(&sess));
                                if (cd == Codec::Google) {
                                        auto *ge                   = static_cast<Codecs::Google::Encoder *>(enc.get());
                                        ge->blockDocs              = GN;
                                        ge->skiplistStep           = GS;
                                        ge->skiplistEntryCountdown = countdown[i];
                                }
                                auto &P = parts[i];
                                enc->begin_term();
                                synth_term(ndocs, i + 1, min_df, seed, [&](uint32_t doc, uint32_t freq, uint64_t y) {
                                        if (doc < doc_lo || doc > doc_hi)
                                                return;
                                        enc->begin_document(doc);
                                        if (with_hits) {
                                                uint32_t pos{0};
                                                for (uint32_t h = 0; h < freq; ++h) {
                                                        pos += synth_pos_step(y, h);
                                                        enc->new_hit(pos);
                                                }
                                        } else {
                                                for (uint32_t h = 0; h < freq; ++h)
                                                        enc->new_hit(h + 1);
                                        }
                                        P.hitsCnt += freq;
                                        enc->end_document();
                                });
                                enc->end_term(&P.t);
                                P.index.swap(sess.indexOut);
                                P.hits.swap(sess.positionsOut);
                        } catch (...) {
                                failed.store(true);
                        }
                }
        };
        std::vector<std::thread> ths;
        for (int i = 1; i < threads; ++i)
                ths.emplace_back(worker);
        worker();
        for (auto &t : ths)
                t.join();
        if (failed.load())
                return TRN_ERR_FORMAT;
        uint64_t ib{0}, hb{0};
        for (auto &p : parts) {
                ib += p.index.size();
                hb += p.hits.size();
        }
        if (ib >= (1ull << 32) || hb >= (1ull << 32))
                return TRN_ERR_CAPACITY; // range32_t limit of one IndexSource (codecs.h:17-55)
        auto s   = new trn_synth();
        s->codec = cd;
        s->index.resize(ib);
        s->hits.resize(hb);
        s->terms.resize(nterms);
        uint64_t io{0}, ho{0};
        for (uint32_t i = 0; i < nterms; ++i) {
                auto &p = parts[i];
                std::memcpy(s->index.data() + io, p.index.data(), p.index.size());
                if (cd == Codec::Lucene) {
                        // the chunk header's first u32 is the term's absolute offset into hits.data (lucene_codec.cpp:178)
                        const uint32_t v   = uint32_t(ho);
                        s->index[io]       = uint8_t(v);
                        s->index[io + 1]   = uint8_t(v >> 8);
                        s->index[io + 2]   = uint8_t(v >> 16);
                        s->index[io + 3]   = uint8_t(v >> 24);
                        if (!p.hits.empty())
                                std::memcpy(s->hits.data() + ho, p.hits.data(), p.hits.size());
                }
                s->terms[i].documents = p.t.documents;
                s->terms[i].chunk_off = uint32_t(io);
                s->terms[i].chunk_len = p.t.size;
                s->sumHits += p.hitsCnt;
                io += p.index.size();
                ho += p.hits.size();
                std::vector<uint8_t>().swap(p.index);
                std::vector<uint8_t>().swap(p.hits);
        }
        *out = s;
        return TRN_OK;
}
extern "C" void trn_synth_destroy(trn_synth *s) {
        delete s;
}
extern "C" int trn_synth_index(trn_synth *s, const uint8_t **index, uint64_t *nbytes) {
        if (!s || !index || !nbytes)
                return TRN_ERR_ARG;
        *index  = s->index.data();
        *nbytes = s->index.size();
        return TRN_OK;
}
extern "C" int trn_synth_hits(trn_synth *s, const uint8_t **hits, uint64_t *nbytes) {
        if (!s || !hits || !nbytes)
                return TRN_ERR_ARG;
        *hits   = s->hits.data();
        *nbytes = s->hits.size();
        return TRN_OK;
}
extern "C" int trn_synth_terms(trn_synth *s, const trn_term **terms, uint32_t *nterms) {
        if (!s || !terms || !nterms)
                return TRN_ERR_ARG;
        *terms  = s->terms.data();
        *nterms = uint32_t(s->terms.size());
        return TRN_OK;
}
extern "C" uint64_t trn_synth_sum_hits(trn_synth *s) {
        return s ? s->sumHits : 0;
}
extern "C" int trn_synth_postings(uint32_t ndocs, uint32_t rank, uint32_t min_df, uint64_t seed, uint32_t *docids, uint32_t *freqs, uint32_t cap, uint32_t *n) {
        if (!ndocs || !rank || !n)
                return TRN_ERR_ARG;
        uint32_t k{0};
        synth_term(ndocs, rank, min_df, seed, [&](uint32_t doc, uint32_t freq, uint64_t) {
                if (k < cap) {
                        if (docids)
                                docids[k] = doc;
                        if (freqs)
                                freqs[k] = freq;
                }
                ++k;
        });
        *n = k;
        return TRN_OK;
}
extern "C" int trn_synth_positions(uint32_t ndocs, uint32_t rank, uint32_t min_df, uint64_t seed, uint32_t *positions, uint64_t cap, uint64_t *n) {
        if (!ndocs || !rank || !n)
                return TRN_ERR_ARG;
        uint64_t k{0};
        synth_term(ndocs, rank, min_df, seed, [&](uint32_t, uint32_t freq, uint64_t y) {
                uint32_t pos{0};
                for (uint32_t h = 0; h < freq; ++h) {
                        pos += synth_pos_step(y, h);
                        if (k < cap && positions)
                                positions[k] = pos;
                        ++k;
                }
        });
        *n = k;
        return TRN_OK;
}

// =================================================================================================== BM25 weights
extern "C" double trn_bm25_idf(uint32_t doc_freq, uint64_t docs_cnt) {
        // similarity.h:179-181: std::log(1 + (docsCnt - docFreq + 0.5f) / (docFreq + 0.5f)), evaluated in float
        const float a = float(uint64_t(docs_cnt - doc_freq)) + 0.5f;
        const float b = float(doc_freq) + 0.5f;
        const float q = a / b;
        return double(std::log(1.0f + q));
}
extern "C" float trn_bm25_score(double idf, uint16_t freq) {
        const float f = float(freq);
        return float(idf * double(f) / double(f + 1.2f));
}

// =================================================================================================== query front-end
namespace {
struct Ast {
        int                  kind; // TRN_NODE_*
        uint32_t             term{0};
        std::vector<int>     kids;
};

struct Parser {
        const char *                                     p, *e;
        const std::unordered_map<std::string, uint32_t> &dict;
        std::vector<Ast>                                 nodes;
        std::string                                      err;

        enum Op { NONE, AND, OR, NOT };
        static int prio(Op o) {
                // queries.cpp:11-27: STRICT_AND / AND / NOT = 8, OR = 7
                return o == OR ? 7 : (o == NONE ? 0 : 8);
        }
        void ws() {
                while (p < e && (*p == ' ' || *p == '\t' || *p == '\n'))
                        ++p;
        }
        static bool isterm(char c) {
                return std::isalnum(static_cast<unsigned char>(c)) || c == '_' || c == ':';
        }
        bool keyword(const char *kw, size_t n) const {
                if (size_t(e - p) < n || std::strncmp(p, kw, n))
                        return false;
                if (p + n == e)
                        return true;
                const char c = p[n];
                return c == ' ' || c == '\t' || c == '(' || c == ')' || c == '-' || c == '+' || c == '.';
        }
        // peeks the operator at the cursor; *len = bytes to consume
        Op peek(size_t *len) {
                ws();
                *len = 0;
                if (p >= e || *p == ')' || *p == '>' || *p == ']' || *p == ',')
                        return NONE;
                if (keyword("AND", 3)) {
                        *len = 3;
                        return AND;
                }
                if (keyword("OR", 2)) {
                        *len = 2;
                        return OR;
                }
                if (keyword("NOT", 3)) {
                        *len = 3;
                        return NOT;
                }
                if (*p == '|') {
                        size_t n = 0;
                        while (p + n < e && p[n] == '|')
                                ++n;
                        *len = n;
                        return OR;
                }
                if (*p == '-' && p + 1 < e && std::isalnum(static_cast<unsigned char>(p[1]))) {
                        *len = 1;
                        return NOT;
                }
                if (isterm(*p) || *p == '(' || *p == '<' || *p == '[' || *p == '"')
                        return AND; // juxtaposition
                return NONE;
        }
        int add(int kind) {
                nodes.push_back(Ast{kind});
                return int(nodes.size()) - 1;
        }
        int depth{0}; // nesting of ( ) [ ] < >: bounded, the parser (and the passes after it) recurse once per level
        struct DepthGuard {
                int &d;
                explicit DepthGuard(int &x) : d{x} { ++d; }
                ~DepthGuard() { --d; }
        };
        int unary() {
                DepthGuard guard(depth);
                if (depth > 200) {
                        err = "expression nested too deeply";
                        return -1;
                }
                ws();
                if (p < e && *p == '<') {
                        // const-true expression (ast_parser::Flags::ParseConstTrueExpr, queries.cpp:378-396): matches like `true`, and, next to
                        // a conjunction operand, only contributes its score -> DocsSetIterators::Optional (exec.cpp:370-377)
                        ++p;
                        const int x = subexpr(255);
                        if (x < 0)
                                return -1;
                        ws();
                        if (p >= e || *p != '>') {
                                err = "expected '>'";
                                return -1;
                        }
                        ++p;
                        const int c   = add(kConstTrue);
                        nodes[c].kids = {x};
                        return c;
                }
                if (p < e && *p == '"') {
                        // "a b c" (parse_phrase_or_token, queries.cpp:70-121): a phrase keeps its terms in order and never de-duplicates them;
                        // one term in quotes is just the term
                        ++p;
                        const int ph = add(TRN_NODE_PHRASE);
                        for (;;) {
                                ws();
                                if (p >= e) {
                                        err = "unterminated phrase";
                                        return -1;
                                }
                                if (*p == '"') {
                                        ++p;
                                        break;
                                }
                                const char *b = p;
                                while (p < e && isterm(*p))
                                        ++p;
                                if (p == b) { // the reference skips characters it cannot tokenise inside a phrase
                                        ++p;
                                        continue;
                                }
                                if (nodes[ph].kids.size() >= 16) // Limits::MaxPhraseSize: the rest is silently ignored (queries.cpp:93-98)
                                        continue;
                                const std::string name(b, p);
                                const int         x  = add(TRN_NODE_TERM);
                                const auto        it = dict.find(name);
                                nodes[x].term        = it == dict.end() ? kEmptyTerm : it->second;
                                nodes[ph].kids.push_back(x);
                        }
                        if (nodes[ph].kids.empty()) {
                                err = "empty phrase";
                                return -1;
                        }
                        if (nodes[ph].kids.size() == 1)
                                return nodes[ph].kids[0];
                        return ph;
                }
                if (p < e && *p == '[') {
                        // [e1, e2, ...] (ast_parser::Flags::ParseMatchSomeExpr, queries.cpp:424-450): ast_node::Type::MatchSome with min = 1; the
                        // application raises match_some.min afterwards (trn_qnode.term of the TRN_NODE_SOME node)
                        ++p;
                        const int s = add(TRN_NODE_SOME);
                        nodes[s].term = 1;
                        for (;;) {
                                const int x = subexpr(255);
                                if (x < 0)
                                        return -1;
                                nodes[s].kids.push_back(x);
                                ws();
                                if (p < e && *p == ',') {
                                        ++p;
                                        continue;
                                }
                                if (p < e && *p == ']') {
                                        ++p;
                                        break;
                                }
                                err = "expected ',' or ']'";
                                return -1;
                        }
                        return s;
                }
                if (p < e && *p == '(') {
                        ++p;
                        const int x = subexpr(255);
                        if (x < 0)
                                return -1;
                        ws();
                        if (p >= e || *p != ')') {
                                err = "expected ')'";
                                return -1;
                        }
                        ++p;
                        return x;
                }
                const char *b = p;
                while (p < e && isterm(*p))
                        ++p;
                if (p == b) {
                        err = "expected a term";
                        return -1;
                }
                const std::string name(b, p);
                if (name == "AND" || name == "OR" || name == "NOT") {
                        err = "operator where a term was expected";
                        return -1;
                }
                const int  x  = add(TRN_NODE_TERM);
                const auto it = dict.find(name);
                nodes[x].term = it == dict.end() ? kEmptyTerm : it->second;
                return x;
        }
        // precedence climbing exactly as parse_subexpr (queries.cpp:477-520): continue while prio(op) < limit, rhs = subexpr(prio(op)),
        // which makes OR bind tighter than AND/NOT and equal priorities left-associative
        int subexpr(int limit) {
                int cur = unary();
                if (cur < 0)
                        return -1;
                for (;;) {
                        size_t   len;
                        const Op op = peek(&len);
                        if (op == NONE || prio(op) >= limit)
                                break;
                        p += len;
                        const int v = subexpr(prio(op));
                        if (v < 0)
                                return -1;
                        if (nodes.size() > 8192) { // the passes below recurse along operator chains; the plan format ends at 65535 nodes anyway
                                err = "query too large";
                                return -1;
                        }
                        const int kind = op == AND ? TRN_NODE_AND : (op == OR ? TRN_NODE_OR : TRN_NODE_NOT);
                        const int x    = add(kind);
                        nodes[x].kids  = {cur, v};
                        cur            = x;
                }
                return cur;
        }
};

// flatten chains of the same associative operator (build_iterator exec.cpp:328-400) and drop duplicate term operands
void flatten_dedup(std::vector<Ast> &n, int i) {
        std::vector<int> ded;
        for (int k : n[i].kids) {
                bool dup{false};
                if (n[k].kind == TRN_NODE_TERM)
                        for (int j : ded)
                                if (n[j].kind == TRN_NODE_TERM && n[j].term == n[k].term)
                                        dup = true;
                if (!dup)
                        ded.push_back(k);
        }
        n[i].kids = ded;
}

// pass 1: merge chains of the same associative operator (build_iterator exec.cpp:328-400) and drop duplicate term operands
void merge_chains(std::vector<Ast> &n, int i) {
        if (n[i].kind == TRN_NODE_TERM)
                return;
        for (int k : n[i].kids)
                merge_chains(n, k);
        if (n[i].kind == TRN_NODE_AND || n[i].kind == TRN_NODE_OR) {
                std::vector<int> out;
                for (int k : n[i].kids) {
                        if (n[k].kind == n[i].kind)
                                out.insert(out.end(), n[k].kids.begin(), n[k].kids.end());
                        else
                                out.push_back(k);
                }
                n[i].kids = out;
                flatten_dedup(n, i);
        }
}

// pass 2: conjunction operands wrapped in <...> become the optional side of an Optional whose main side is the rest of the chain
void convert_consttrue(std::vector<Ast> &n, int i) {
        if (n[i].kind == TRN_NODE_TERM)
                return;
        {
                const std::vector<int> kids = n[i].kids; // n may grow (reallocate) below
                for (int k : kids)
                        convert_consttrue(n, k);
        }
        if (n[i].kind != TRN_NODE_AND)
                return;
        std::vector<int> mains, opts;
        for (int k : n[i].kids)
                (n[k].kind == kConstTrue ? opts : mains).push_back(k);
        if (opts.empty() || mains.empty())
                return;
        int mainNode;
        if (mains.size() == 1)
                mainNode = mains[0];
        else {
                n.push_back(Ast{TRN_NODE_AND, 0, mains});
                mainNode = int(n.size()) - 1;
        }
        // several <...> operands of one conjunction are merged by the reference's compiler into ONE const-true expression over
        // their conjunction ([<foo> AND <bar>] => [<foo,bar>], compilation_ctx.cpp:371-385)
        int optExpr = n[opts[0]].kids[0];
        if (opts.size() > 1) {
                std::vector<int> es;
                for (int o : opts)
                        es.push_back(n[o].kids[0]);
                n.push_back(Ast{TRN_NODE_AND, 0, es});
                optExpr = int(n.size()) - 1;
                merge_chains(n, optExpr);
        }
        n[i].kind = TRN_NODE_OPTIONAL;
        n[i].kids = {mainNode, optExpr};
}

void flatten(std::vector<Ast> &n, int i) {
        merge_chains(n, i);
        convert_consttrue(n, i);
}
} // namespace

// == the terms dictionary an IndexSource resolves query tokens through (IndexSource::resolve_term_ctx, index_source.h:118):
// name -> term id, built ONCE and owned by the caller as an explicit handle.
struct trn_dict {
        std::unordered_map<std::string, uint32_t> map;
};

extern "C" int trn_dict_create(const char *const *names, uint32_t nterms, trn_dict **out) {
        if (!out || (nterms && !names))
                return TRN_ERR_ARG;
        try {
                auto d = std::make_unique<trn_dict>();
                d->map.reserve(size_t(nterms) * 2);
                for (uint32_t i = 0; i < nterms; ++i) {
                        if (!names[i])
                                return TRN_ERR_ARG;
                        d->map.emplace(names[i], i); // first occurrence wins, like a dictionary lookup would
                }
                *out = d.release();
                return TRN_OK;
        } catch (...) {
                return TRN_ERR_CAPACITY;
        }
}
extern "C" void trn_dict_destroy(trn_dict *d) {
        delete d;
}

static int parse_query_impl(const char *text, const std::unordered_map<std::string, uint32_t> &dict, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root,
                            char *err, size_t errcap);

extern "C" int trn_parse_query_dict(const char *text, const trn_dict *dict, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root, char *err,
                                    size_t errcap) {
        if (!text || !dict || !nodes || !nnodes || !root)
                return TRN_ERR_ARG;
        return parse_query_impl(text, dict->map, nodes, cap, nnodes, root, err, errcap);
}

// convenience form: resolves through a names array; the map is rebuilt on every call (nothing is cached across calls — a caller that
// parses many queries against one vocabulary creates a trn_dict once)
extern "C" int trn_parse_query(const char *text, const char *const *names, uint32_t nterms, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root,
                               char *err, size_t errcap) {
        if (!text || !nodes || !nnodes || !root || (nterms && !names))
                return TRN_ERR_ARG;
        std::unordered_map<std::string, uint32_t> dict;
        try {
                dict.reserve(size_t(nterms) * 2);
                for (uint32_t i = 0; i < nterms; ++i)
                        if (names[i])
                                dict.emplace(names[i], i);
        } catch (...) {
                return TRN_ERR_CAPACITY;
        }
        return parse_query_impl(text, dict, nodes, cap, nnodes, root, err, errcap);
}

static int parse_query_impl(const char *text, const std::unordered_map<std::string, uint32_t> &dict, trn_qnode *nodes, uint32_t cap, uint32_t *nnodes, uint32_t *root,
                            char *err, size_t errcap) {
        auto seterr = [&](const std::string &m) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return TRN_ERR_PARSE;
        };
        Parser ps{text, text + std::strlen(text), dict, {}, {}};
        const int r = ps.subexpr(255);
        if (r < 0)
                return seterr(ps.err);
        ps.ws();
        if (ps.p != ps.e)
                return seterr("trailing input at offset " + std::to_string(ps.p - text));
        flatten(ps.nodes, r);
        // single-child AND/OR after de-duplication collapse to the child
        // single-operand AND/OR and const-true wrappers that did not end up beside a conjunction operand collapse to their child
        auto collapse = [&](int x) {
                while (ps.nodes[x].kind != TRN_NODE_TERM && ps.nodes[x].kids.size() == 1 &&
                       (ps.nodes[x].kind == TRN_NODE_AND || ps.nodes[x].kind == TRN_NODE_OR || ps.nodes[x].kind == kConstTrue ||
                        ps.nodes[x].kind == TRN_NODE_SOME)) // [x] == x: compilation_ctx.cpp:786-789 (the parser always yields min = 1)
                        x = ps.nodes[x].kids[0];
                return x;
        };
        int rr = collapse(r);
        // emit breadth-first so that children are contiguous and follow their parent
        std::vector<int> order{rr};
        std::vector<trn_qnode> out;
        out.reserve(32);
        out.push_back(trn_qnode{});
        for (size_t qi = 0; qi < order.size(); ++qi) {
                const Ast &A = ps.nodes[order[qi]];
                trn_qnode  q;
                std::memset(&q, 0, sizeof(q));
                q.kind = uint8_t(A.kind);
                if (A.kind == TRN_NODE_TERM)
                        q.term = A.term;
                else {
                        if (A.kind == TRN_NODE_SOME)
                                q.term = A.term; // min-should-match
                        std::vector<int> kids;
                        for (int k : A.kids) {
                                kids.push_back(collapse(k));
                        }
                        if (kids.size() > 255 || out.size() + kids.size() > 65535)
                                return seterr("query too large");
                        q.nchildren   = uint8_t(kids.size());
                        q.first_child = uint16_t(out.size());
                        for (int k : kids) {
                                order.push_back(k);
                                out.push_back(trn_qnode{});
                        }
                }
                out[qi] = q;
        }
        if (out.size() > cap)
                return seterr("node buffer too small");
        std::memcpy(nodes, out.data(), out.size() * sizeof(trn_qnode));
        *nnodes = uint32_t(out.size());
        *root   = 0;
        return TRN_OK;
}

// ------------------------------------------------------------------------------------------------ pipeline plan (host only: tests, tooling)
// The launches trn_exec_batch would split a DocumentsOnly / SCORED_ALL batch into (csrc/chunkplan.h — the same function the engine calls), from
// the quantities it knows before the first launch.  sizes[] receives the queries per launch (at most cap), *n their number, *single_call
// whether the batch takes the one-call form.
extern "C" int trn_debug_chunk_plan(uint32_t nq, int topk, uint64_t est_postings, uint64_t leaves, uint32_t max_chunks, uint64_t chunk_postings, int rule_sqrt,
                                    int taper, double tail_ms, double tail_tree_ms, uint64_t hint_bytes, uint64_t hint_postings, int hint_same_shape,
                                    uint32_t *sizes, uint32_t cap, uint32_t *n, int *single_call) {
        if (!n || !single_call || (cap && !sizes))
                return TRN_ERR_ARG;
        ChunkPlanIn in;
        in.nq              = nq;
        in.topk            = topk != 0;
        in.est_postings    = est_postings;
        in.leaves          = leaves;
        in.max_chunks      = max_chunks;
        in.chunk_postings  = chunk_postings;
        in.rule_sqrt       = rule_sqrt != 0;
        in.taper           = taper != 0;
        in.tail_ms         = tail_ms;
        in.tail_tree_ms    = tail_tree_ms;
        in.hint_bytes      = hint_bytes;
        in.hint_postings   = hint_postings;
        in.hint_same_shape = hint_same_shape != 0;
        const ChunkPlan P  = plan_chunks(in);
        *n                 = uint32_t(P.sizes.size());
        *single_call       = P.single_call ? 1 : 0;
        for (uint32_t i = 0; i < *n && i < cap; ++i)
                sizes[i] = P.sizes[i];
        return *n <= cap ? TRN_OK : TRN_ERR_CAPACITY;
}

// ------------------------------------------------------------------------------------------------ result replay
// == the MatchesProxy::process / consider(docid_t) stream of one query (docset_spans.h:14-21, matches.h:149-171), from either result form
template <class F> static int replay_query(const trn_result *r, uint32_t q, F &&f) {
        if (!r || q >= r->nq || !r->offsets)
                return TRN_ERR_ARG;
        if (r->docids) { // TRN_MODE_DOCS_ONLY / SCORED_*: plain docIDs
                for (uint64_t i = r->offsets[q]; i < r->offsets[q + 1]; ++i)
                        if (f(r->docids[i]))
                                return TRN_OK;
                return TRN_OK;
        }
        if (!r->words || !r->item_desc || !r->qitems)
                return r->offsets[q] == r->offsets[q + 1] ? TRN_OK : TRN_ERR_ARG;
        const trn_qitems &Q = r->qitems[q];
        const uint32_t *  w = r->words + r->offsets[q];
        for (uint32_t j = 0; j < Q.nitems; ++j) {
                const uint32_t d = r->item_desc[Q.item_base + j], n = d & 0x3fffffffu, enc = d >> 30;
                if (!n)
                        continue;
                const uint32_t base = (Q.tile_lo + j) << Q.tile_shift;
                if (enc == TRN_ENC_U32) {
                        for (uint32_t i = 0; i < n; ++i)
                                if (f(w[i]))
                                        return TRN_OK;
                        w += n;
                } else if (enc == TRN_ENC_U16) {
                        for (uint32_t i = 0; i < n; ++i)
                                if (f(base + ((w[i >> 1] >> ((i & 1u) * 16u)) & 0xffffu)))
                                        return TRN_OK;
                        w += (n + 1u) >> 1;
                } else if (enc == TRN_ENC_BITMAP) {
                        const uint32_t nw = (1u << Q.tile_shift) >> 5;
                        for (uint32_t k = 0; k < nw; ++k) {
                                uint32_t x = w[k];
                                while (x) {
                                        const uint32_t b = uint32_t(__builtin_ctz(x));
                                        x &= x - 1u;
                                        if (f(base + 32u * k + b))
                                                return TRN_OK;
                                }
                        }
                        w += nw;
                } else { // TRN_ENC_U8B
                        const uint32_t nbk = (1u << Q.tile_shift) >> 8, nwords = (nbk + n + 3u) >> 2;
                        if (!nbk || w + nwords > r->words + r->offsets[q + 1])
                                return TRN_ERR_FORMAT;
                        const uint8_t *cnt = reinterpret_cast<const uint8_t *>(w), *off = cnt + nbk;
                        uint32_t       k{0};
                        for (uint32_t b = 0; b < nbk; ++b) {
                                if (k + cnt[b] > n)
                                        return TRN_ERR_FORMAT;
                                for (uint32_t i = 0; i < cnt[b]; ++i)
                                        if (f(base + 256u * b + off[k++]))
                                                return TRN_OK;
                        }
                        if (k != n)
                                return TRN_ERR_FORMAT; // the buckets must add up to the item's documents
                        w += nwords;
                }
        }
        return w == r->words + r->offsets[q + 1] ? TRN_OK : TRN_ERR_FORMAT; // the segments must add up to the query's words
}

extern "C" int trn_result_for_each(const trn_result *r, uint32_t q, trn_consider_fn fn, void *ctx) {
        if (!fn)
                return TRN_ERR_ARG;
        return replay_query(r, q, [&](uint32_t id) { return fn(ctx, id) != 0; });
}

extern "C" int trn_result_decode(const trn_result *r, uint32_t q, uint32_t *out, uint64_t cap, uint64_t *n) {
        if (!n || (!out && cap))
                return TRN_ERR_ARG;
        uint64_t  k{0};
        bool      over{false};
        const int rc = replay_query(r, q, [&](uint32_t id) {
                if (k < cap)
                        out[k] = id;
                else
                        over = true;
                ++k;
                return false;
        });
        *n = k;
        if (rc != TRN_OK)
                return rc;
        return over ? TRN_ERR_CAPACITY : TRN_OK;
}
