// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's query-token intersections (intersect.h:25-37), built by oracle/build_intersect.sh into
// oracle/_ref/libtrinity_ref_isect.so together with the reference's own intersect.cpp (compiled in place), against the reference objects of
// libtrinity_ref.so:
//   * single source: intersect(0, tokens, src, registry) over an in-memory source of either codec (index bytes, LUCENE hits.data, terms), with
//     masked documents
//   * collection:    intersect(0, tokens, collection) over segment directories written by the reference's SegmentIndexSession
// Tokens are given as names; group g is names[offsets[g] .. offsets[g + 1]).  Only tests/ and scripts/ load it.
#include "google_codec.h"
#include "intersect.h"
#include "lucene_codec.h"
#include "segment_index_source.h"
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
                term_index_ctx resolve_term_ctx(const str8_t term) override {
                        auto it = terms.find(std::string(term.data(), term.size()));
                        return it == terms.end() ? term_index_ctx{} : it->second;
                }
                Codecs::Decoder *new_postings_decoder(const str8_t, const term_index_ctx ctx) override {
                        return ap->new_decoder(ctx);
                }
                field_statistics default_field_stats() override {
                        return {};
                }
                bool index_empty() const override {
                        return false;
                }
        };

        struct Handle {
                std::vector<uint8_t>                    index, hits;
                std::unique_ptr<Codecs::AccessProxy>    ap;
                std::unique_ptr<IndexSourcesCollection> col;
                IndexSource *                           src{nullptr};
                std::vector<std::pair<uint64_t, uint32_t>> last;
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

        std::vector<std::unordered_set<str8_t>> token_groups(uint32_t ngroups, const uint32_t *offsets, const char *const *names) {
                std::vector<std::unordered_set<str8_t>> tokens(ngroups);
                for (uint32_t g = 0; g < ngroups; ++g)
                        for (uint32_t i = offsets[g]; i < offsets[g + 1]; ++i)
                                tokens[g].insert(str8_t(names[i], uint8_t(strlen(names[i]))));
                return tokens;
        }
} // namespace

extern "C" {
const char *tisect_last_error() {
        return g_err.c_str();
}

void *tisect_source(int codec, const uint8_t *index, uint64_t n, const uint8_t *hits, uint64_t nh, const char *const *names, const uint32_t *docs, const uint32_t *off, const uint32_t *len,
                    uint32_t nterms) {
        auto x = new Handle();
        if (guarded([&] {
                    x->index.assign(index, index + n);
                    if (hits && nh)
                            x->hits.assign(hits, hits + nh);
                    if (codec == 0)
                            x->ap.reset(new Codecs::Google::AccessProxy("/tmp", x->index.data()));
                    else
                            x->ap.reset(new Codecs::Lucene::AccessProxy("/tmp", x->index.data(), x->hits.empty() ? (const uint8_t *)"" : x->hits.data()));
                    auto s = new Src();
                    s->ap  = x->ap.get();
                    for (uint32_t i = 0; i < nterms; ++i)
                            s->terms.emplace(names[i], term_index_ctx(docs[i], range32_t{off[i], len[i]}));
                    x->src = s;
                    x->col.reset(new IndexSourcesCollection());
                    x->col->insert(s);
                    s->Release();
                    x->col->commit();
            })) {
                delete x;
                return nullptr;
        }
        return x;
}

// segment directories, scanned newest generation first (index_source.cpp:3-30)
void *tisect_collection(const char *const *dirs, uint32_t n) {
        auto x = new Handle();
        if (guarded([&] {
                    x->col.reset(new IndexSourcesCollection());
                    for (uint32_t i = 0; i < n; ++i) {
                            auto seg = new SegmentIndexSource(dirs[i]);
                            x->col->insert(seg);
                            seg->Release();
                    }
                    x->col->commit();
            })) {
                delete x;
                return nullptr;
        }
        return x;
}

void tisect_free(void *h) {
        delete static_cast<Handle *>(h);
}

// intersect(0, tokens, src, registry of `masked`); returns the number of {mask, count} pairs (tisect_last), -1 on error
int64_t tisect_run(void *h, uint32_t ngroups, const uint32_t *offsets, const char *const *names, const uint32_t *masked, uint32_t nmasked) {
        auto    x = static_cast<Handle *>(h);
        int64_t n{-1};
        guarded([&] {
                const auto           tokens = token_groups(ngroups, offsets, names);
                std::vector<docid_t> v(masked, masked + nmasked);
                IOBuffer             packed;
                pack_updates(v, &packed);
                auto ud  = unpack_updates({reinterpret_cast<const uint8_t *>(packed.data()), uint32_t(packed.size())});
                auto reg = masked_documents_registry::make(&ud, 1);
                x->last  = intersect(0, tokens, x->src, reg.get());
                n        = int64_t(x->last.size());
        });
        return n;
}

// intersect(0, tokens, collection)
int64_t tisect_run_collection(void *h, uint32_t ngroups, const uint32_t *offsets, const char *const *names) {
        auto    x = static_cast<Handle *>(h);
        int64_t n{-1};
        guarded([&] {
                x->last = intersect(0, token_groups(ngroups, offsets, names), x->col.get());
                n       = int64_t(x->last.size());
        });
        return n;
}

void tisect_last(void *h, uint64_t *masks, uint32_t *counts) {
        auto x = static_cast<Handle *>(h);
        for (size_t i = 0; i < x->last.size(); ++i) {
                masks[i]  = x->last[i].first;
                counts[i] = x->last[i].second;
        }
}
}
