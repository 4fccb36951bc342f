// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's default exec mode (exec_query with no ExecFlags: consider(const matched_document &)), built by
// oracle/build_matches.sh into oracle/_ref/libtrinity_ref_matches.so against the reference objects of libtrinity_ref.so:
//   * in-memory indexes built through the reference Encoders WITH payloads (codecs.h:195 new_hit(pos, payload))
//   * exec_query(flags 0), optionally with a masked_documents_registry, recording per match the matched terms (queryCtx->term.token),
//     hits->freq and hits->all[0 .. freq)
// Only tests/ and scripts/ load it.
#include "exec.h"
#include "google_codec.h"
#include "lucene_codec.h"
#include <cstring>
#include <string>
#include <unordered_map>
#include <vector>

using namespace Trinity;

namespace {
        thread_local std::string g_err;

        struct Src final : public IndexSource {
                Codecs::AccessProxy *                           ap{nullptr};
                std::unordered_map<std::string, term_index_ctx> terms;
                field_statistics                                fs;
                term_index_ctx resolve_term_ctx(const str8_t term) override {
                        auto it = terms.find(std::string(term.data(), term.size()));
                        return it == terms.end() ? term_index_ctx{} : it->second;
                }
                Codecs::Decoder *new_postings_decoder(const str8_t, const term_index_ctx ctx) override {
                        return ap->new_decoder(ctx);
                }
                field_statistics default_field_stats() override {
                        return fs;
                }
                bool index_empty() const override {
                        return false;
                }
        };

        struct Idx {
                int                                   codec{0};
                std::unique_ptr<Codecs::IndexSession> sess;
                std::unique_ptr<Codecs::Encoder>      enc;
                std::vector<uint8_t>                  index, hits;
                std::vector<term_index_ctx>           tctx;
                std::vector<std::string>              names;
                std::unordered_map<std::string, uint32_t> ids;
                std::unique_ptr<Codecs::AccessProxy>  ap;
                Src *                                 src{nullptr};
                std::unique_ptr<IndexSourcesCollection> col;
                uint64_t                              sumHits{0};
                // the last exec
                std::vector<uint32_t> docids, term_counts, terms, freqs;
                std::vector<uint64_t> payloads;
                std::vector<uint16_t> pos;
                std::vector<uint8_t>  plen;
                ~Idx() {
                        col.reset();
                }
        };

        struct Recorder final : public MatchedIndexDocumentsFilter {
                Idx *x;
                void consider(const matched_document &m) override {
                        x->docids.push_back(m.id);
                        x->term_counts.push_back(m.matchedTermsCnt);
                        for (uint32_t i = 0; i < m.matchedTermsCnt; ++i) {
                                const auto &mt = m.matchedTerms[i];
                                const auto  tk = mt.queryCtx->term.token;
                                const auto  it = x->ids.find(std::string(tk.data(), tk.size()));
                                x->terms.push_back(it == x->ids.end() ? 0xffffffffu : it->second);
                                x->freqs.push_back(mt.hits->freq);
                                for (uint32_t h = 0; h < mt.hits->freq; ++h) {
                                        x->payloads.push_back(mt.hits->all[h].payload);
                                        x->pos.push_back(mt.hits->all[h].pos);
                                        x->plen.push_back(mt.hits->all[h].payloadLen);
                                }
                        }
                }
        };

        template <typename F>
        int guarded(F &&f) {
                try {
                        f();
                        return 0;
                } catch (const std::exception &e) {
                        g_err = e.what();
                } catch (...) {
                        g_err = "unknown exception";
                }
                return -1;
        }
} // namespace

extern "C" {
const char *trefm_last_error() {
        return g_err.c_str();
}

void *trefm_new(int codec) {
        auto x   = new Idx();
        x->codec = codec;
        if (codec == 0)
                x->sess.reset(new Codecs::Google::IndexSession("/tmp"));
        else
                x->sess.reset(new Codecs::Lucene::IndexSession("/tmp"));
        x->sess->begin();
        x->enc.reset(x->sess->new_encoder());
        return x;
}

void trefm_free(void *h) {
        delete static_cast<Idx *>(h);
}

// positions: every hit's absolute position, documents concatenated (sum(freqs) entries); plens[i] payload bytes of hit i (0..8), its bytes
// the low plens[i] bytes of payloads[i] (little-endian)
int trefm_add_term(void *h, const char *name, const uint32_t *docids, const uint32_t *freqs, uint32_t n, const uint32_t *positions, const uint8_t *plens,
                   const uint64_t *payloads) {
        auto x = static_cast<Idx *>(h);
        int  idx{-1};
        if (guarded([&] {
                    term_index_ctx t;
                    size_t         pi{0};
                    x->enc->begin_term();
                    for (uint32_t i = 0; i < n; ++i) {
                            x->enc->begin_document(docids[i]);
                            for (uint32_t k = 0; k < freqs[i]; ++k, ++pi) {
                                    uint8_t b[8];
                                    std::memcpy(b, &payloads[pi], 8);
                                    x->enc->new_hit(positions[pi], {b, plens[pi]});
                            }
                            x->sumHits += freqs[i];
                            x->enc->end_document();
                    }
                    x->enc->end_term(&t);
                    idx = int(x->tctx.size());
                    x->tctx.push_back(t);
                    x->ids.emplace(name, uint32_t(idx));
                    x->names.emplace_back(name);
            }))
                return -1;
        return idx;
}

int trefm_finish(void *h, uint64_t docsCnt) {
        auto x = static_cast<Idx *>(h);
        return guarded([&] {
                x->index.assign((const uint8_t *)x->sess->indexOut.data(), (const uint8_t *)x->sess->indexOut.data() + x->sess->indexOut.size());
                if (x->codec == 1) {
                        auto ls = static_cast<Codecs::Lucene::IndexSession *>(x->sess.get());
                        x->hits.assign((const uint8_t *)ls->positionsOut.data(), (const uint8_t *)ls->positionsOut.data() + ls->positionsOut.size());
                }
                x->enc.reset();
                x->sess.reset();
                if (x->codec == 0)
                        x->ap.reset(new Codecs::Google::AccessProxy("/tmp", x->index.data()));
                else
                        x->ap.reset(new Codecs::Lucene::AccessProxy("/tmp", x->index.data(), x->hits.empty() ? (const uint8_t *)"" : x->hits.data()));
                auto s = new Src();
                x->src = s;
                s->ap  = x->ap.get();
                uint64_t sumDocs{0};
                for (size_t i = 0; i < x->names.size(); ++i) {
                        s->terms.emplace(x->names[i], x->tctx[i]);
                        sumDocs += x->tctx[i].documents;
                }
                s->fs.docsCnt      = docsCnt;
                s->fs.sumTermsDocs = sumDocs;
                s->fs.totalTerms   = x->names.size();
                s->fs.sumTermHits  = x->sumHits;
                x->col.reset(new IndexSourcesCollection());
                x->col->insert(s);
                s->Release();
                x->col->commit();
        });
}

uint64_t trefm_index_size(void *h) {
        return static_cast<Idx *>(h)->index.size();
}
const uint8_t *trefm_index_data(void *h) {
        return static_cast<Idx *>(h)->index.data();
}
uint64_t trefm_hits_size(void *h) {
        return static_cast<Idx *>(h)->hits.size();
}
const uint8_t *trefm_hits_data(void *h) {
        return static_cast<Idx *>(h)->hits.data();
}
void trefm_term(void *h, uint32_t idx, uint32_t *docs, uint32_t *off, uint32_t *len) {
        const auto &t = static_cast<Idx *>(h)->tctx[idx];
        *docs         = t.documents;
        *off          = t.indexChunk.offset;
        *len          = t.indexChunk.size();
}

static void set_min(ast_node *n, uint16_t m) {
        if (!n)
                return;
        switch (n->type) {
                case ast_node::Type::BinOp:
                        set_min(n->binop.lhs, m);
                        set_min(n->binop.rhs, m);
                        break;
                case ast_node::Type::UnaryOp:
                        set_min(n->unaryop.expr, m);
                        break;
                case ast_node::Type::ConstTrueExpr:
                        set_min(n->expr, m);
                        break;
                case ast_node::Type::MatchSome:
                        n->match_some.min = m;
                        for (size_t i = 0; i < n->match_some.size; ++i)
                                set_min(n->match_some.nodes[i], m);
                        break;
                default:
                        break;
        }
}

// exec_query(flags 0); minMatch != 0: match_some.min of every MatchSome group; masked: the masked_documents_registry's docIDs.
// Returns the number of matches; trefm_last gives what was recorded.
int64_t trefm_exec_matches(void *h, const char *q, uint32_t parserFlags, uint32_t minMatch, const uint32_t *masked, uint32_t nmasked) {
        auto    x = static_cast<Idx *>(h);
        int64_t n{-1};
        guarded([&] {
                for (auto *v : {&x->docids, &x->term_counts, &x->terms, &x->freqs})
                        v->clear();
                x->payloads.clear();
                x->pos.clear();
                x->plen.clear();
                query qq(str32_t(q, strlen(q)), default_token_parser_impl, parserFlags);
                if (minMatch)
                        set_min(qq.root, uint16_t(minMatch));
                Recorder             rec;
                std::vector<docid_t> v(masked, masked + nmasked);
                IOBuffer             packed;
                rec.x = x;
                pack_updates(v, &packed);
                auto ud  = unpack_updates({reinterpret_cast<const uint8_t *>(packed.data()), uint32_t(packed.size())});
                auto reg = masked_documents_registry::make(&ud, 1);
                exec_query(qq, x->src, reg.get(), &rec, nullptr, 0u);
                n = int64_t(x->docids.size());
        });
        return n;
}

void trefm_last(void *h, const uint32_t **docids, const uint32_t **term_counts, const uint32_t **terms, const uint32_t **freqs, const uint64_t **payloads,
                const uint16_t **pos, const uint8_t **plen, uint64_t *nterms, uint64_t *nhits) {
        auto x       = static_cast<Idx *>(h);
        *docids      = x->docids.data();
        *term_counts = x->term_counts.data();
        *terms       = x->terms.data();
        *freqs       = x->freqs.data();
        *payloads    = x->payloads.data();
        *pos         = x->pos.data();
        *plen        = x->plen.data();
        *nterms      = x->terms.size();
        *nhits       = x->pos.size();
}
}
