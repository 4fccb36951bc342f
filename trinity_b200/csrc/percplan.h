// The percolator's registration planner (trn_percolator_register, engine.cu): per query a post-order program over presence bits and an
// anchor cover, and the term -> anchored-queries index the device walks (percolate.cuh).  A pure function of the query trees, the vocabulary
// size and the term costs — so it is pinned on the CPU (trn_debug_percolator_plan, tests/test_percolate_cpu.py).  Host only.
//
// An anchor cover of a query is a set of terms such that every document the query matches holds at least one of them (DESIGN.md §4):
//   TERM: the term.  PHRASE: its cheapest term.  AND: the cheapest cover among its operands.  OR: the union of its operands' covers.
//   SOME (min k): of the m operands that can match, the union of the covers of the cheapest m - k + 1.  NOT: its required side's.
//   OPTIONAL: its main side's.
// Two other outcomes are kept apart: NEVER (no document can match: a term outside the vocabulary, k > m, an AND over such an operand) and
// UNANCHORED (a match may hold none of the query's terms); a NEVER operand drops out of an OR / SOME, an UNANCHORED one makes them
// unanchored and never supplies an AND's cover.  Cost = the sum of term_cost over the cover (1 per term without costs); ties go to the
// lexicographically smaller sorted cover, then to the earlier operand.
#pragma once
#include "../../include/trinity_b200.h"
#include "device_types.h"
#include "planner.h"
#include <algorithm>
#include <cstdint>
#include <string>
#include <tuple>
#include <vector>

namespace trn {

enum : uint8_t { PERC_ANCHORED = 0, PERC_UNANCHORED = 1, PERC_NEVER = 2 };

struct PercPlan {
        std::vector<PercQuery> queries;
        std::vector<uint8_t>   status; // per query: PERC_ANCHORED / PERC_UNANCHORED / PERC_NEVER
        std::vector<PercOp>    ops;
        std::vector<uint32_t>  phrase_terms, covers;
        std::vector<uint32_t>  csr_off; // nterms + 1
        std::vector<PercEntry> csr;
        std::vector<uint32_t>  unanchored;
        std::vector<uint32_t>  npt; // per query: its phrase terms (consecutive in phrase_terms, in the order of its PHRASE ops)
        uint32_t               never{0};
};

namespace percplan_detail {
struct Cover {
        uint8_t               kind{PERC_NEVER};
        std::vector<uint32_t> terms; // ascending
        uint64_t              cost{0};
};
inline bool cheaper(const Cover &a, const Cover &b) {
        return std::tie(a.cost, a.terms) < std::tie(b.cost, b.terms);
}

struct Builder {
        const trn_qnode *n;
        const uint32_t * cost;
        PercPlan &       P;
        uint32_t         depth{0}, max_depth{0};

        uint64_t c(uint32_t t) const {
                return cost ? cost[t] : 1u;
        }
        void push(const PercOp &o, uint32_t pops) {
                P.ops.push_back(o);
                depth = depth - pops + 1u;
                max_depth = std::max(max_depth, depth);
        }
        // emits node i's program (post order) and returns its cover
        Cover node(uint32_t i) {
                const trn_qnode &X = n[i];
                Cover            r;
                if (X.kind == TRN_NODE_TERM) {
                        if (X.term == kEmptyTerm) {
                                push(PercOp{PERC_CONST, 0, 0, 0}, 0);
                                return r;
                        }
                        push(PercOp{PERC_TERM, 0, 0, X.term}, 0);
                        r.kind  = PERC_ANCHORED;
                        r.terms = {X.term};
                        r.cost  = c(X.term);
                        return r;
                }
                if (X.kind == TRN_NODE_PHRASE) {
                        uint32_t best = 0;
                        for (uint32_t k = 0; k < X.nchildren; ++k) {
                                const uint32_t t = n[X.first_child + k].term, b = n[X.first_child + best].term;
                                if (t == kEmptyTerm) {
                                        push(PercOp{PERC_CONST, 0, 0, 0}, 0);
                                        return r;
                                }
                                if (std::make_tuple(c(t), t) < std::make_tuple(c(b), b))
                                        best = k;
                        }
                        const uint32_t at = uint32_t(P.phrase_terms.size());
                        for (uint32_t k = 0; k < X.nchildren; ++k)
                                P.phrase_terms.push_back(n[X.first_child + k].term);
                        push(PercOp{PERC_PHRASE, X.nchildren, uint16_t(best), at}, 0);
                        const uint32_t t = n[X.first_child + best].term;
                        r.kind           = PERC_ANCHORED;
                        r.terms          = {t};
                        r.cost           = c(t);
                        return r;
                }
                std::vector<Cover> kids;
                for (uint32_t k = 0; k < X.nchildren; ++k)
                        kids.push_back(node(X.first_child + k));
                const uint8_t nk = X.nchildren;
                switch (X.kind) {
                case TRN_NODE_NOT:
                        push(PercOp{PERC_NOT, nk, 0, 0}, nk);
                        return kids[0];
                case TRN_NODE_OPTIONAL:
                        push(PercOp{PERC_OPT, nk, 0, 0}, nk);
                        return kids[0];
                case TRN_NODE_AND: {
                        push(PercOp{PERC_AND, nk, 0, 0}, nk);
                        const Cover *best = nullptr;
                        for (const Cover &k : kids) {
                                if (k.kind == PERC_NEVER)
                                        return r;
                                if (k.kind == PERC_ANCHORED && (!best || cheaper(k, *best)))
                                        best = &k;
                        }
                        if (!best)
                                r.kind = PERC_UNANCHORED;
                        return best ? *best : r;
                }
                default: break;
                }
                // OR / SOME: the covers of the `need` cheapest operands that can match
                std::vector<uint32_t> live;
                for (uint32_t k = 0; k < nk; ++k)
                        if (kids[k].kind != PERC_NEVER)
                                live.push_back(k);
                size_t need = live.size();
                if (X.kind == TRN_NODE_SOME) {
                        push(PercOp{PERC_SOME, nk, uint16_t(std::min<uint32_t>(X.term, 256u)), 0}, nk);
                        if (X.term < 1 || X.term > live.size())
                                return r;
                        need = live.size() - X.term + 1u;
                } else {
                        push(PercOp{PERC_OR, nk, 0, 0}, nk);
                        if (live.empty())
                                return r;
                }
                std::stable_sort(live.begin(), live.end(), [&](uint32_t a, uint32_t b) {
                        const bool ua = kids[a].kind != PERC_ANCHORED, ub = kids[b].kind != PERC_ANCHORED;
                        return ua != ub ? ub : cheaper(kids[a], kids[b]);
                });
                for (size_t j = 0; j < need; ++j) {
                        const Cover &k = kids[live[j]];
                        if (k.kind != PERC_ANCHORED) {
                                r.kind = PERC_UNANCHORED;
                                r.terms.clear();
                                r.cost = 0;
                                return r;
                        }
                        r.terms.insert(r.terms.end(), k.terms.begin(), k.terms.end());
                }
                std::sort(r.terms.begin(), r.terms.end());
                r.terms.erase(std::unique(r.terms.begin(), r.terms.end()), r.terms.end());
                r.kind = PERC_ANCHORED;
                for (const uint32_t t : r.terms)
                        r.cost += c(t);
                return r;
        }
};
} // namespace percplan_detail

// The per-query part of the plan: queries[0 .. nq) get the ids first_id .. first_id + nq - 1 and their programs, covers and statuses are
// appended to P (offsets relative to P's own arrays; P.unanchored holds ids).  A query's program, cover and status depend only on its tree,
// nterms and term_cost, so planning a set in slices and concatenating them gives what planning it whole gives (trn_percolator_add).
// Returns TRN_OK, or TRN_ERR_ARG (a malformed tree, a phrase of more than 16 terms, a term id >= nterms other than kEmptyTerm) /
// TRN_ERR_UNSUPPORTED (a program that needs more than kPercStack pending operands) / TRN_ERR_CAPACITY (2^32 anchor entries), naming the
// query by its index in `queries` in err.
inline int perc_plan_queries(const trn_query *queries, uint32_t nq, uint32_t first_id, uint32_t nterms, const uint32_t *term_cost, PercPlan &P,
                             std::string &err) {
        const size_t q0 = P.queries.size();
        P.queries.resize(q0 + nq);
        P.status.resize(q0 + nq);
        P.npt.resize(q0 + nq);
        for (uint32_t q = 0; q < nq; ++q) {
                const trn_query &Q   = queries[q];
                const std::string who = "query " + std::to_string(q) + ": ";
                std::string      e;
                bool             unsupported{false}, has_phrase{false};
                if (!Q.nodes || !Q.nnodes || !validate_plan(Q.nodes, Q.nnodes, Q.root, nterms, true, e, unsupported, has_phrase)) {
                        err = who + (Q.nodes && Q.nnodes ? e : std::string("no nodes"));
                        return TRN_ERR_ARG;
                }
                percplan_detail::Builder b{Q.nodes, term_cost, P};
                PercQuery &              R  = P.queries[q0 + q];
                const size_t             pt = P.phrase_terms.size();
                R.op_begin                  = uint32_t(P.ops.size());
                percplan_detail::Cover c    = b.node(Q.root);
                R.nops                      = uint32_t(P.ops.size()) - R.op_begin;
                if (b.max_depth > kPercStack) {
                        err = who + "its program needs " + std::to_string(b.max_depth) + " pending operands (at most " + std::to_string(kPercStack) + ")";
                        return TRN_ERR_UNSUPPORTED;
                }
                P.status[q0 + q] = c.kind;
                P.npt[q0 + q]    = uint32_t(P.phrase_terms.size() - pt);
                R.cover_begin    = uint32_t(P.covers.size());
                R.ncover         = uint32_t(c.terms.size());
                P.covers.insert(P.covers.end(), c.terms.begin(), c.terms.end());
                if (c.kind == PERC_UNANCHORED)
                        P.unanchored.push_back(first_id + q);
                else if (c.kind == PERC_NEVER)
                        ++P.never;
                if (P.covers.size() >= (1ull << 32)) {
                        err = who + "the registry's anchor entries reach 2^32";
                        return TRN_ERR_CAPACITY;
                }
        }
        return TRN_OK;
}

// The whole registration: the per-query part over every query (ids 0 .. nq - 1), then the term -> (query, ordinal) CSR, ascending query id
// within every term.  The refusals of perc_plan_queries.
inline int perc_plan(const trn_query *queries, uint32_t nq, uint32_t nterms, const uint32_t *term_cost, PercPlan &P, std::string &err) {
        P = PercPlan{};
        if (const int rc = perc_plan_queries(queries, nq, 0, nterms, term_cost, P, err))
                return rc;
        P.csr_off.assign(size_t(nterms) + 1u, 0u);
        for (const uint32_t t : P.covers)
                ++P.csr_off[t + 1u];
        for (uint32_t t = 0; t < nterms; ++t)
                P.csr_off[t + 1u] += P.csr_off[t];
        P.csr.resize(P.covers.size());
        std::vector<uint32_t> at(P.csr_off.begin(), P.csr_off.end() - 1);
        for (uint32_t q = 0; q < nq; ++q)
                for (uint32_t j = 0; j < P.queries[q].ncover; ++j)
                        P.csr[at[P.covers[P.queries[q].cover_begin + j]]++] = PercEntry{q, j};
        return TRN_OK;
}

} // namespace trn
