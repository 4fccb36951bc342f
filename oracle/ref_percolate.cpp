// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's percolator (percolator.h, percolator.cpp), built by oracle/build_percolate.sh into
// oracle/_ref/libtrinity_ref_perc.so together with the reference's own percolator.cpp (compiled in place), against the reference objects of
// libtrinity_ref.so (compile_query, group_execnodes, the query parser).
//   * queries: each text is parsed with Trinity::query and the given ast_parser flags (8 = ParseConstTrueExpr, 16 = ParseMatchSomeExpr), its
//     MatchSome groups get match_some.min = the given min when non-zero (as tref_exec3 does), and becomes a percolator_query
//   * documents: token ids into a vocabulary of names (0xffffffff: a token outside it); token i sits at position i + 1
//   * the proxy: match_term(t) = the document holds the vocabulary id of term_by_index(t); match_phrase(t0..tk) = at some position p the
//     tokens at p .. p + k are the vocabulary ids of t0 .. tk.  A query term outside the vocabulary never matches.
// Only tests/ and scripts/ load it.
#include "percolator.h"
#include <cstring>
#include <memory>
#include <string>
#include <unordered_map>
#include <unordered_set>
#include <vector>

using namespace Trinity;

namespace {
        thread_local std::string g_err;
        constexpr uint32_t       kOov = 0xffffffffu;

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

        void set_match_some_min(ast_node *n, uint16_t m) {
                if (!n)
                        return;
                switch (n->type) {
                        case ast_node::Type::BinOp:
                                set_match_some_min(n->binop.lhs, m);
                                set_match_some_min(n->binop.rhs, m);
                                break;
                        case ast_node::Type::UnaryOp:
                                set_match_some_min(n->unaryop.expr, m);
                                break;
                        case ast_node::Type::ConstTrueExpr:
                                set_match_some_min(n->expr, m);
                                break;
                        case ast_node::Type::MatchSome:
                                n->match_some.min = m;
                                for (size_t i = 0; i < n->match_some.size; ++i)
                                        set_match_some_min(n->match_some.nodes[i], m);
                                break;
                        default:
                                break;
                }
        }

        struct Query {
                std::unique_ptr<percolator_query> pq;
                std::vector<uint32_t>             vocab; // local term index - 1 -> vocabulary id (kOov outside it)
        };

        struct Proxy final : percolator_document_proxy {
                const Query *                q{nullptr};
                const uint32_t *             tok{nullptr};
                uint32_t                     n{0};
                std::unordered_set<uint32_t> held;

                bool match_term(const uint16_t t) override {
                        const uint32_t v = q->vocab[t - 1];
                        return v != kOov && held.count(v);
                }
                bool match_phrase(const uint16_t *ts, const uint16_t cnt) override {
                        for (uint32_t k = 0; k < cnt; ++k)
                                if (q->vocab[ts[k] - 1] == kOov)
                                        return false;
                        for (uint32_t p = 0; p + cnt <= n; ++p) {
                                uint32_t k = 0;
                                while (k < cnt && tok[p + k] == q->vocab[ts[k] - 1])
                                        ++k;
                                if (k == cnt)
                                        return true;
                        }
                        return false;
                }
        };

        struct Handle {
                std::vector<Query>    queries;
                std::vector<uint64_t> offsets;
                std::vector<uint32_t> ids;
        };
} // namespace

extern "C" {
const char *tperc_last_error() {
        return g_err.c_str();
}

// queries[i] parsed with flags[i] and min[i]; the vocabulary resolves its terms.  nullptr on error (tperc_last_error).
void *tperc_new(const char *const *queries, const uint32_t *flags, const uint32_t *mins, uint32_t nq, const char *const *vocab, uint32_t nvocab) {
        auto x = new Handle();
        if (guarded([&] {
                    std::unordered_map<std::string, uint32_t> dict;
                    for (uint32_t i = 0; i < nvocab; ++i)
                            dict.emplace(vocab[i], i);
                    x->queries.resize(nq);
                    for (uint32_t i = 0; i < nq; ++i) {
                            query qq(str32_t(queries[i], strlen(queries[i])), default_token_parser_impl, flags[i]);
                            if (mins[i])
                                    set_match_some_min(qq.root, uint16_t(mins[i]));
                            Query &Q = x->queries[i];
                            Q.pq.reset(new percolator_query(qq));
                            for (const auto &t : Q.pq->distinct_terms()) {
                                    const auto it = dict.find(std::string(t.data(), t.size()));
                                    Q.vocab.push_back(it == dict.end() ? kOov : it->second);
                            }
                    }
            })) {
                delete x;
                return nullptr;
        }
        return x;
}

void tperc_free(void *h) {
        delete static_cast<Handle *>(h);
}

// every document against every query (what the reference offers: one match() per pair); returns the number of matches, -1 on error
int64_t tperc_run(void *h, const uint64_t *doc_offsets, const uint32_t *tokens, uint32_t ndocs) {
        auto    x = static_cast<Handle *>(h);
        int64_t n{-1};
        guarded([&] {
                x->offsets.assign(1, 0);
                x->ids.clear();
                Proxy px;
                for (uint32_t d = 0; d < ndocs; ++d) {
                        px.tok = tokens + doc_offsets[d];
                        px.n   = uint32_t(doc_offsets[d + 1] - doc_offsets[d]);
                        px.held.clear();
                        for (uint32_t i = 0; i < px.n; ++i)
                                if (px.tok[i] != kOov)
                                        px.held.insert(px.tok[i]);
                        for (uint32_t q = 0; q < x->queries.size(); ++q) {
                                px.q = &x->queries[q];
                                if (x->queries[q].pq->match(px))
                                        x->ids.push_back(q);
                        }
                        x->offsets.push_back(x->ids.size());
                }
                n = int64_t(x->ids.size());
        });
        return n;
}

// the last run's result: offsets[ndocs + 1], ids[total]
void tperc_last(void *h, uint64_t *offsets, uint32_t *ids) {
        auto x = static_cast<Handle *>(h);
        std::memcpy(offsets, x->offsets.data(), x->offsets.size() * 8);
        std::memcpy(ids, x->ids.data(), x->ids.size() * 4);
}
}
