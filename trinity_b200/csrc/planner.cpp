// The batch planner (planner.h) and the plan compiler it runs per query.  The compiler mirrors the host side of the reference's exec
// path: queryexec_ctx::build_iterator + build_span (exec.cpp:253-505), operator tree -> per-tile step program, including the
// IteratorScorer combination rules of docset_iterators_scorers.cpp:8-242 (which leaves contribute to a document's score is structural;
// see Compiler::node()).
#include "planner.h"
#include <algorithm>
#include <cmath>
#include <cstdlib>
#include <cstring>

using namespace trn;

namespace {
struct Range {
        uint32_t lo{1}, hi{0}; // inclusive docIDs; empty when lo > hi
        bool     empty() const {
                return lo > hi;
        }
};

// every node has at most one parent: a plan is a TREE (a node shared by several parents would make the recursive passes — cost, range,
// bound, truth tables — revisit it once per path, exponentially often in a hostile plan)
static bool plan_is_tree(const trn_qnode *n, uint32_t nn, uint32_t root) {
        std::vector<uint8_t> seen(nn, 0);
        if (root < nn)
                seen[root] = 1;
        for (uint32_t i = 0; i < nn; ++i) {
                if (n[i].kind == TRN_NODE_TERM)
                        continue;
                for (uint32_t k = 0; k < n[i].nchildren; ++k) {
                        const uint32_t c = uint32_t(n[i].first_child) + k;
                        if (c >= nn || seen[c])
                                return false;
                        seen[c] = 1;
                }
        }
        return true;
}

// children follow their parents in the node array (checked by validate()), so one forward pass yields every node's depth; the
// compiler and the truth-table builder recurse once per level
static bool plan_depth_ok(const trn_qnode *n, uint32_t nn) {
        std::vector<uint8_t> depth(nn, 0);
        for (uint32_t i = 0; i < nn; ++i) {
                if (n[i].kind == TRN_NODE_TERM)
                        continue;
                if (depth[i] >= 64)
                        return false;
                for (uint32_t k = 0; k < n[i].nchildren; ++k) {
                        const uint32_t c = uint32_t(n[i].first_child) + k;
                        if (c > i && c < nn)
                                depth[c] = uint8_t(std::max<int>(depth[c], depth[i] + 1));
                }
        }
        return true;
}
} // namespace

bool trn::validate_plan(const trn_qnode *n, uint32_t nn, uint32_t root, uint32_t nterms, bool allow_phrase, std::string &err, bool &unsupported, bool &has_phrase) {
        if (root >= nn) {
                err = "root out of range";
                return false;
        }
        if (!plan_depth_ok(n, nn)) {
                err = "query tree deeper than 64 levels";
                return false;
        }
        for (uint32_t i = 0; i < nn; ++i) {
                if (n[i].kind == TRN_NODE_TERM) {
                        if (n[i].term != kEmptyTerm && n[i].term >= nterms) {
                                err = "term id out of range";
                                return false;
                        }
                } else if (n[i].kind == TRN_NODE_PHRASE) {
                        if (!allow_phrase) {
                                err         = "phrase nodes need the positions (materialize_hits): a LUCENE source executes them once its hits.data has been uploaded (trn_upload_hits)";
                                unsupported = true;
                                return false;
                        }
                        if (n[i].nchildren < 2 || n[i].nchildren > 16 || n[i].first_child <= i || uint32_t(n[i].first_child) + n[i].nchildren > nn) {
                                err = "a phrase holds 2..16 terms behind it in the node array";
                                return false;
                        }
                        for (uint32_t k = 0; k < n[i].nchildren; ++k)
                                if (n[n[i].first_child + k].kind != TRN_NODE_TERM) {
                                        err = "the children of a phrase are terms";
                                        return false;
                                }
                        has_phrase = true;
                } else if (n[i].kind > TRN_NODE_PHRASE) {
                        err = "unknown node kind";
                        return false;
                } else {
                        // children must come after their parent (guarantees an acyclic tree)
                        if (n[i].nchildren == 0 || n[i].first_child <= i || uint32_t(n[i].first_child) + n[i].nchildren > nn) {
                                err = "children must follow their parent in the node array";
                                return false;
                        }
                }
        }
        if (!plan_is_tree(n, nn, root)) {
                err = "a node is referenced by more than one parent (a plan is a tree)";
                return false;
        }
        return true;
}

namespace {
struct Compiler {
        const trn_qnode *           n;
        uint32_t                    nn;
        const std::vector<DevTerm> &terms;
        bool                        scored;
        uint32_t                    root;
        std::vector<DevStep> &      steps;
        uint32_t                    next_slot{0};
        uint64_t                    postings{0}, bytes{0};
        struct Deferred {
                uint32_t              term;
                double                idf;
                std::vector<uint8_t> cond;
                int                   phrase{-1}; // >= 0: node index of a phrase (its position check is repeated under the condition's mask)
        };
        std::vector<Deferred> deferred;
        std::string           err;
        bool                  reference_quirks{true};
        bool                  unsupported{false};
        bool                  allow_phrase{false}; // the caller's kernels execute OP_PHRASE (GOOGLE codec: inline hits)
        bool                  has_phrase{false};

        Compiler(const trn_qnode *nodes, uint32_t cnt, const std::vector<DevTerm> &t, bool sc, uint32_t r, std::vector<DevStep> &s)
            : n{nodes}, nn{cnt}, terms{t}, scored{sc}, root{r}, steps{s} {
        }

        // Slots: in DocumentsOnly plans a child's bitmap is dead once it has been combined into its parent, so its slot is handed out
        // again (scored plans keep every slot: the deferred scoring pass reads branch bitmaps at the end).  Fewer live slots = less
        // shared memory per worker = more resident warps (with one slot per node the 8-term trees left few warps resident per SM).
        std::vector<uint32_t> free_slots;
        int alloc_slot() {
                if (!scored && !free_slots.empty()) {
                        const auto it = std::min_element(free_slots.begin(), free_slots.end());
                        const int  v  = int(*it);
                        free_slots.erase(it);
                        return v;
                }
                if (next_slot >= 14) {
                        err = "query needs more than 14 docset slots";
                        return -1;
                }
                return int(next_slot++);
        }
        void release_slot(uint32_t s) {
                if (!scored)
                        free_slots.push_back(s);
        }

        bool is_leaf(uint32_t i) const {
                return n[i].kind == TRN_NODE_TERM;
        }
        bool is_phrase(uint32_t i) const {
                return n[i].kind == TRN_NODE_PHRASE;
        }
        // the conjunction of a phrase's distinct terms into slot `tmp` (rarest first), then the position check in place (phrase.cuh)
        void phrase_steps(uint32_t i, uint32_t tmp, bool score) {
                const auto &          X = n[i];
                std::vector<uint32_t> t(X.nchildren);
                double                idfsum{0};
                bool                  anyEmpty{false};
                for (uint32_t j = 0; j < X.nchildren; ++j) {
                        t[j] = n[X.first_child + j].term;
                        idfsum += n[X.first_child + j].weight;
                        anyEmpty |= t[j] == kEmptyTerm || terms[t[j]].documents == 0;
                }
                if (anyEmpty) { // a phrase with an unknown term matches nothing
                        push(OP_CLEAR, 0, tmp, 0, 0, 0, 0);
                        return;
                }
                std::vector<uint32_t> distinct(t);
                std::sort(distinct.begin(), distinct.end());
                distinct.erase(std::unique(distinct.begin(), distinct.end()), distinct.end());
                std::stable_sort(distinct.begin(), distinct.end(), [&](uint32_t a, uint32_t b) { return terms[a].documents < terms[b].documents; });
                bool first{true};
                for (auto term : distinct) {
                        postings += terms[term].documents;
                        bytes += terms[term].chunk_len;
                        push(OP_LEAF, first ? M_SET : M_AND, tmp, 0, 0, term, 0);
                        first = false;
                }
                push(OP_PHRASE, uint8_t(X.nchildren), tmp, 0, score ? F_SCORE : 0, 0, idfsum);
                for (uint32_t j = 0; j < X.nchildren; j += 4) { // four term ids per operand step, in phrase order
                        DevStep a;
                        std::memset(&a, 0, sizeof(a));
                        a.op   = OP_ARG;
                        a.term = t[j];
                        a.pad2 = j + 1 < X.nchildren ? t[j + 1] : 0u;
                        const uint64_t hi = uint64_t(j + 2 < X.nchildren ? t[j + 2] : 0u) | (uint64_t(j + 3 < X.nchildren ? t[j + 3] : 0u) << 32);
                        std::memcpy(&a.idf, &hi, 8);
                        steps.push_back(a);
                }
        }
        // a phrase operand combined into dst with `mode` (== leaf() for a term); scores score(matchCnt, sum idf) where it holds
        bool phrase_leaf(uint32_t i, uint8_t mode, uint32_t dst, bool scoring, const std::vector<uint8_t> &cond, uint8_t extraFlags) {
                const bool wantScore = scored && scoring;
                if (mode == M_NONE && !wantScore)
                        return true; // nothing to do in this pass
                const bool immediate = wantScore && cond.empty();
                if (wantScore && !immediate)
                        deferred.push_back({0, 0.0, cond, int(i)});
                if (mode == M_NONE && !immediate)
                        return true; // the deferred pass does it all
                const int tmp = alloc_slot();
                if (tmp < 0)
                        return false;
                phrase_steps(i, uint32_t(tmp), immediate);
                if (mode != M_NONE)
                        push(OP_SLOT, mode, dst, uint32_t(tmp), extraFlags, 0, 0);
                release_slot(uint32_t(tmp));
                return true;
        }
        uint32_t df(uint32_t i) const {
                const auto t = n[i].term;
                return t == kEmptyTerm ? 0u : terms[t].documents;
        }
        void push(uint8_t op, uint8_t mode, uint32_t dst, uint32_t src, uint8_t flags, uint32_t term, double idf) {
                DevStep s;
                std::memset(&s, 0, sizeof(s));
                s.op    = op;
                s.mode  = mode;
                s.dst   = uint8_t(dst);
                s.src   = uint8_t(src);
                s.flags = flags;
                s.term  = term;
                s.idf   = idf;
                steps.push_back(s);
        }
        void account(uint32_t i) {
                const auto t = n[i].term;
                if (t != kEmptyTerm) {
                        postings += terms[t].documents;
                        bytes += terms[t].chunk_len;
                }
        }
        // leaf combined into dst with `mode`; scoring per the structural rules
        void leaf(uint32_t i, uint8_t mode, uint32_t dst, bool scoring, const std::vector<uint8_t> &cond, uint8_t extraFlags) {
                account(i);
                uint8_t flags = extraFlags;
                if (scored && scoring) {
                        if (cond.empty())
                                flags |= F_SCORE;
                        else
                                deferred.push_back({n[i].term, n[i].weight, cond});
                }
                if (mode == M_NONE && !(flags & F_SCORE))
                        return; // nothing to do in this pass
                push(OP_LEAF, mode, dst, 0, flags, n[i].term, n[i].weight);
        }

        // compiles internal node i into its own slot; returns the slot
        int node(uint32_t i, bool scoring, const std::vector<uint8_t> &cond) {
                const int sAlloc = alloc_slot();
                if (sAlloc < 0)
                        return -1;
                const uint32_t s    = uint32_t(sAlloc);
                const auto &   X    = n[i];
                const bool     isRoot = i == root;
                if (X.nchildren == 0 || uint32_t(X.first_child) + X.nchildren > nn) {
                        err = "operator node without (valid) children";
                        return -1;
                }
                std::vector<uint32_t> kids(X.nchildren);
                for (uint32_t c = 0; c < X.nchildren; ++c)
                        kids[c] = X.first_child + c;
                auto child_cond = [&](uint32_t slotOfChild) {
                        auto v = cond;
                        v.push_back(uint8_t(slotOfChild));
                        return v;
                };
                switch (X.kind) {
                        case TRN_NODE_AND: {
                                // leaves first, rarest first (== prepare_tree's df sort exec.cpp:154-170 and reorder_execnodes :216)
                                std::stable_sort(kids.begin(), kids.end(), [&](uint32_t a, uint32_t b) {
                                        const bool la = is_leaf(a), lb = is_leaf(b);
                                        if (la != lb)
                                                return la;
                                        if (la)
                                                return df(a) < df(b);
                                        return false;
                                });
                                bool first{true};
                                for (auto c : kids) {
                                        const uint8_t fl = isRoot ? F_BREAK_IF_EMPTY : 0;
                                        if (is_leaf(c))
                                                leaf(c, first ? M_SET : M_AND, s, scoring, cond, fl);
                                        else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, first ? M_SET : M_AND, s, scoring, cond, fl))
                                                        return -1;
                                        } else {
                                                const int cs = node(c, scoring, cond);
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, first ? M_SET : M_AND, s, uint32_t(cs), fl, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                        first = false;
                                }
                        } break;
                        case TRN_NODE_OR: {
                                push(OP_CLEAR, 0, s, 0, 0, 0, 0);
                                for (auto c : kids) {
                                        if (is_leaf(c))
                                                leaf(c, M_OR, s, scoring, cond, 0);
                                        else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, M_OR, s, scoring, cond, 0))
                                                        return -1;
                                        } else {
                                                // a non-leaf child of a disjunction contributes its score only for documents it matches itself
                                                // (Disjunction scorer sums children positioned on the doc, docset_iterators_scorers.cpp)
                                                const uint32_t willBe = next_slot;
                                                const int      cs     = node(c, scoring, child_cond(willBe));
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, M_OR, s, uint32_t(cs), 0, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                }
                        } break;
                        case TRN_NODE_NOT:
                        case TRN_NODE_OPTIONAL: {
                                if (X.nchildren != 2) {
                                        err = "NOT / OPTIONAL need exactly two children";
                                        return -1;
                                }
                                const uint8_t fl = isRoot ? F_BREAK_IF_EMPTY : 0;
                                if (is_leaf(kids[0]))
                                        leaf(kids[0], M_SET, s, scoring, cond, fl);
                                else if (is_phrase(kids[0])) {
                                        if (!phrase_leaf(kids[0], M_SET, s, scoring, cond, fl))
                                                return -1;
                                } else {
                                        const int cs = node(kids[0], scoring, cond);
                                        if (cs < 0)
                                                return -1;
                                        push(OP_SLOT, M_SET, s, uint32_t(cs), fl, 0, 0);
                                        release_slot(uint32_t(cs));
                                }
                                if (X.kind == TRN_NODE_NOT) {
                                        // Filter: excluded side never scores (docset_iterators_scorers.cpp Filter -> req only)
                                        if (is_leaf(kids[1]))
                                                leaf(kids[1], M_ANDNOT, s, false, cond, 0);
                                        else if (is_phrase(kids[1])) {
                                                if (!phrase_leaf(kids[1], M_ANDNOT, s, false, cond, 0))
                                                        return -1;
                                        } else {
                                                const int cs = node(kids[1], false, cond);
                                                if (cs < 0)
                                                        return -1;
                                                push(OP_SLOT, M_ANDNOT, s, uint32_t(cs), 0, 0, 0);
                                                release_slot(uint32_t(cs));
                                        }
                                } else if (scored && scoring) {
                                        // Optional: main drives; opt only adds its score when it is on the document
                                        if (is_leaf(kids[1]))
                                                leaf(kids[1], M_NONE, s, true, cond, 0);
                                        else if (is_phrase(kids[1])) {
                                                if (!phrase_leaf(kids[1], M_NONE, s, true, cond, 0))
                                                        return -1;
                                        } else {
                                                const uint32_t willBe = next_slot;
                                                if (node(kids[1], true, child_cond(willBe)) < 0)
                                                        return -1;
                                        }
                                } else {
                                        // docs-only: the optional side cannot change the match set, but it is still "touched" by the reference
                                        // (Optional::next advances opt lazily); we do not read it at all.
                                }
                        } break;
                        case TRN_NODE_SOME: {
                                // DisjunctionSome (docset_iterators.cpp:679-811): every child is evaluated into a bitmap of its own and added to a
                                // bit-sliced saturating counter (one bitmap per counter bit); the node matches where the counter reaches `min`.
                                // A child scores only where it matches AND the node matches (Wrapper::iterator_score sums the lead list).
                                const uint32_t m = X.term;
                                if (m == 0 || m > 15) {
                                        err = "SOME: min-should-match must be in 1..15";
                                        return -1;
                                }
                                uint32_t k = 1;
                                while (((1u << k) - 1u) < m)
                                        ++k;
                                if (next_slot + k + 1 > 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                const uint32_t p0 = next_slot;
                                next_slot += k;
                                const uint32_t t = next_slot++; // shared by the leaf children
                                for (uint32_t j = 0; j < k; ++j)
                                        push(OP_CLEAR, 0, p0 + j, 0, 0, 0, 0);
                                for (auto c : kids) {
                                        uint32_t src;
                                        if (is_leaf(c)) {
                                                leaf(c, M_SET, t, scoring, child_cond(s), 0);
                                                src = t;
                                        } else if (is_phrase(c)) {
                                                if (!phrase_leaf(c, M_SET, t, scoring, child_cond(s), 0))
                                                        return -1;
                                                src = t;
                                        } else {
                                                auto cc = child_cond(s);
                                                cc.push_back(uint8_t(next_slot)); // the child's own slot
                                                const int cs = node(c, scoring, cc);
                                                if (cs < 0)
                                                        return -1;
                                                src = uint32_t(cs);
                                        }
                                        push(OP_COUNT_ADD, uint8_t(k), p0, src, 0, 0, 0);
                                        if (src != t)
                                                release_slot(src);
                                }
                                push(OP_COUNT_GE, uint8_t(k), s, p0, 0, m, 0);
                                for (uint32_t j = 0; j < k; ++j)
                                        release_slot(p0 + j);
                                release_slot(t);
                        } break;
                        default:
                                err = "unknown node kind";
                                return -1;
                }
                return int(s);
        }

        Range range(uint32_t i) const {
                const auto &X = n[i];
                Range       r;
                if (X.kind == TRN_NODE_TERM) {
                        if (X.term != kEmptyTerm && terms[X.term].documents) {
                                r.lo = terms[X.term].first_doc;
                                r.hi = terms[X.term].last_doc;
                        }
                        return r;
                }
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return range(X.first_child);
                const bool conj = X.kind == TRN_NODE_AND || X.kind == TRN_NODE_PHRASE; // a phrase needs all of its terms
                bool       first{true};
                for (uint32_t c = 0; c < X.nchildren; ++c) {
                        const Range cr = range(X.first_child + c);
                        if (conj) {
                                if (cr.empty())
                                        return Range{};
                                if (first)
                                        r = cr;
                                else {
                                        r.lo = std::max(r.lo, cr.lo);
                                        r.hi = std::min(r.hi, cr.hi);
                                        if (r.empty())
                                                return Range{};
                                }
                                first = false;
                        } else {
                                if (cr.empty())
                                        continue;
                                if (first)
                                        r = cr;
                                else {
                                        r.lo = std::min(r.lo, cr.lo);
                                        r.hi = std::max(r.hi, cr.hi);
                                }
                                first = false;
                        }
                }
                return r;
        }

        uint64_t bound(uint32_t i) const {
                const auto &X = n[i];
                if (X.kind == TRN_NODE_TERM)
                        return df(i);
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return bound(X.first_child);
                const bool conj = X.kind == TRN_NODE_AND || X.kind == TRN_NODE_PHRASE;
                uint64_t   b    = conj ? ~0ull : 0ull;
                for (uint32_t c = 0; c < X.nchildren; ++c) {
                        const uint64_t cb = bound(X.first_child + c);
                        b                 = conj ? std::min(b, cb) : b + cb;
                }
                return b;
        }

        bool validate() {
                return validate_plan(n, nn, root, uint32_t(terms.size()), allow_phrase, err, unsupported, has_phrase);
        }

        // == DocsSetIterators::cost() (docset_iterators.cpp:10-64); a conjunction's cost is its lead's, which the reference's
        // reordering passes make the cheapest operand
        uint64_t cost(uint32_t i) const {
                const auto &X = n[i];
                if (X.kind == TRN_NODE_TERM)
                        return df(i);
                if (X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL)
                        return cost(X.first_child);
                if (X.kind == TRN_NODE_PHRASE) // docset_iterators.cpp:50-55: cost(its[0]) + UINT32_MAX + UINT16_MAX * size
                        return cost(X.first_child) + 0xffffffffull + 0xffffull * X.nchildren;
                if (X.kind == TRN_NODE_SOME) { // DisjunctionSome::cost_: the (size - min + 1) cheapest children (docset_iterators.cpp:733-742)
                        std::vector<uint64_t> cs;
                        for (uint32_t k = 0; k < X.nchildren; ++k)
                                cs.push_back(cost(X.first_child + k));
                        std::sort(cs.begin(), cs.end());
                        const uint32_t keep = X.nchildren >= X.term ? X.nchildren - X.term + 1u : 0u;
                        uint64_t       c{0};
                        for (uint32_t k = 0; k < keep && k < cs.size(); ++k)
                                c += cs[k];
                        return c;
                }
                uint64_t c = X.kind == TRN_NODE_AND ? ~0ull : 0ull;
                for (uint32_t k = 0; k < X.nchildren; ++k) {
                        const uint64_t cc = cost(X.first_child + k);
                        c                 = X.kind == TRN_NODE_AND ? std::min(c, cc) : c + cc;
                }
                return c;
        }

        // REFERENCE QUIRK, mirrored for drop-in parity: build_span() (exec.cpp:488-501) turns a root Filter whose excluded side is not
        // costlier than its required side into FilteredDocsSetSpan(build_span(req), excl).  When req is a disjunction the inner span is
        // DocsSetSpanForDisjunctions[WithThreshold], whose process() ignores its `min` argument (docset_spans.cpp:98-111,681-694): the
        // excluded documents the outer span stepped over are emitted by the next call anyway, so the exclusion has no effect and the
        // reference returns the plain disjunction.  The same holds through a chain of such root filters.
        void apply_reference_root_filter_quirk() {
                uint32_t cur = root;
                bool     traversed{false};
                while (n[cur].kind == TRN_NODE_NOT && n[cur].nchildren == 2 && cost(n[cur].first_child + 1u) <= cost(n[cur].first_child)) {
                        cur       = n[cur].first_child;
                        traversed = true;
                }
                if (traversed && n[cur].kind == TRN_NODE_OR)
                        root = cur;
        }

        // returns root slot or -1
        int run() {
                if (!validate())
                        return -1;
                if (reference_quirks)
                        apply_reference_root_filter_quirk();
                int rs;
                if (is_leaf(root)) {
                        rs = int(next_slot++);
                        leaf(root, M_SET, uint32_t(rs), true, {}, 0);
                } else if (is_phrase(root)) {
                        rs = int(next_slot++);
                        if (!phrase_leaf(root, M_SET, uint32_t(rs), true, {}, 0))
                                return -1;
                } else
                        rs = node(root, true, {});
                if (rs < 0)
                        return -1;
                // second pass for leaves whose contribution is conditional on a disjunction branch matching
                for (auto &d : deferred) {
                        uint32_t mask = d.cond[0];
                        if (d.cond.size() > 1) {
                                if (next_slot >= 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                mask = next_slot++;
                                push(OP_SLOT, M_SET, mask, d.cond[0], 0, 0, 0);
                                for (size_t j = 1; j < d.cond.size(); ++j)
                                        push(OP_SLOT, M_AND, mask, d.cond[j], 0, 0, 0);
                        }
                        if (d.phrase >= 0) { // the phrase again, restricted to the condition's documents, scoring this time
                                if (next_slot >= 14) {
                                        err = "query needs more than 14 docset slots";
                                        return -1;
                                }
                                const uint32_t tmp = next_slot++;
                                // (phrase_steps starts with SET/CLEAR into tmp; the mask narrows the candidates before the position check)
                                const size_t at = steps.size();
                                phrase_steps(uint32_t(d.phrase), tmp, true);
                                // insert [SLOT AND tmp, mask] in front of the OP_PHRASE step
                                for (size_t z = at; z < steps.size(); ++z)
                                        if (steps[z].op == OP_PHRASE) {
                                                DevStep a;
                                                std::memset(&a, 0, sizeof(a));
                                                a.op   = OP_SLOT;
                                                a.mode = M_AND;
                                                a.dst  = uint8_t(tmp);
                                                a.src  = uint8_t(mask);
                                                steps.insert(steps.begin() + z, a);
                                                break;
                                        }
                                continue;
                        }
                        push(OP_LEAFSCORE, M_NONE, 0, mask, 0, d.term, d.idf);
                }
                return rs;
        }
};
} // namespace

// Truth vector of a query subtree over its (<= 8) distinct terms: bit `a` (0..255) = value of the node when exactly the terms whose
// bit is set in `a` are present (bit j of `a` = term tv[j]).  Bitwise evaluation: one 256-bit operation per node.
struct TruthVec {
        uint64_t w[4];
};
static TruthVec truth_vector(const trn_qnode *nodes, uint32_t i, const uint32_t *tv, uint32_t n) {
        static const uint64_t kPat[6] = {0xaaaaaaaaaaaaaaaaull, 0xccccccccccccccccull, 0xf0f0f0f0f0f0f0f0ull, 0xff00ff00ff00ff00ull, 0xffff0000ffff0000ull, 0xffffffff00000000ull};
        const auto &X = nodes[i];
        TruthVec    v{{0, 0, 0, 0}};
        if (X.kind == TRN_NODE_TERM) {
                for (uint32_t j = 0; j < n; ++j)
                        if (tv[j] == X.term) {
                                for (int q = 0; q < 4; ++q)
                                        v.w[q] = j < 6 ? kPat[j] : (j == 6 ? ((q & 1) ? ~0ull : 0ull) : ((q & 2) ? ~0ull : 0ull));
                                break;
                        }
                return v;
        }
        const uint32_t f = X.first_child;
        if (X.kind == TRN_NODE_SOME) {
                const uint32_t        nk = X.nchildren; // all of them (<= 255)
                std::vector<TruthVec> kids(nk);
                for (uint32_t k = 0; k < nk; ++k)
                        kids[k] = truth_vector(nodes, f + k, tv, n);
                for (uint32_t a = 0; a < 256; ++a) {
                        uint32_t cnt{0};
                        for (uint32_t k = 0; k < nk; ++k)
                                cnt += uint32_t((kids[k].w[a >> 6] >> (a & 63u)) & 1ull);
                        if (cnt >= X.term)
                                v.w[a >> 6] |= 1ull << (a & 63u);
                }
                return v;
        }
        v = truth_vector(nodes, f, tv, n);
        for (uint32_t k = 1; k < X.nchildren; ++k) {
                const TruthVec w = truth_vector(nodes, f + k, tv, n);
                for (int q = 0; q < 4; ++q) {
                        if (X.kind == TRN_NODE_AND) v.w[q] &= w.w[q];
                        else if (X.kind == TRN_NODE_OR) v.w[q] |= w.w[q];
                        else if (X.kind == TRN_NODE_NOT) v.w[q] &= ~w.w[q];
                        // OPTIONAL: the optional side never changes the match set
                }
        }
        return v;
}

// The distinct terms below node `root` (at most 8, in walk order) into tv[0 .. n); kEmptyTerm is skipped, and with `terms` a term without
// postings too.  TRN_ERR_ARG: more than 8 of them or a malformed subtree; TRN_ERR_UNSUPPORTED: a phrase below root.
static int distinct_terms(const trn_qnode *nodes, uint32_t nnodes, uint32_t root, const std::vector<DevTerm> *terms, uint32_t *tv, uint32_t &n) {
        uint32_t stack[64], sp{0};
        n           = 0;
        stack[sp++] = root;
        while (sp) {
                const auto &X = nodes[stack[--sp]];
                if (X.kind == TRN_NODE_TERM) {
                        if (X.term == kEmptyTerm || (terms && !(*terms)[X.term].nblocks))
                                continue;
                        bool seen{false};
                        for (uint32_t j = 0; j < n; ++j)
                                seen |= tv[j] == X.term;
                        if (!seen) {
                                if (n == 8)
                                        return TRN_ERR_ARG;
                                tv[n++] = X.term;
                        }
                } else {
                        if (X.kind == TRN_NODE_PHRASE)
                                return TRN_ERR_UNSUPPORTED;
                        if (X.kind > TRN_NODE_SOME || X.nchildren == 0 || uint32_t(X.first_child) + X.nchildren > nnodes || sp + X.nchildren > 64)
                                return TRN_ERR_ARG;
                        for (uint32_t k = 0; k < X.nchildren; ++k)
                                stack[sp++] = X.first_child + k;
                }
        }
        return TRN_OK;
}

extern "C" int trn_query_truth_table(const trn_qnode *nodes, uint32_t nnodes, uint32_t root, uint32_t *terms, uint32_t *nterms, uint32_t *table, uint32_t *necessary) {
        if (!nodes || !nnodes || root >= nnodes || !terms || !nterms || !table || !necessary)
                return TRN_ERR_ARG;
        for (uint32_t i = 0; i < nnodes; ++i) // same structural rules as the plan compiler: children behind their parent, bounded depth
                if (nodes[i].kind != TRN_NODE_TERM && (nodes[i].nchildren == 0 || nodes[i].first_child <= i || uint32_t(nodes[i].first_child) + nodes[i].nchildren > nnodes))
                        return TRN_ERR_ARG;
        if (!plan_depth_ok(nodes, nnodes) || !plan_is_tree(nodes, nnodes, root))
                return TRN_ERR_ARG;
        uint32_t  n{0};
        const int rc = distinct_terms(nodes, nnodes, root, nullptr, terms, n);
        if (rc != TRN_OK)
                return rc;
        const TruthVec v = truth_vector(nodes, root, terms, n);
        uint32_t       nec{n ? (1u << n) - 1u : 0u};
        for (uint32_t w = 0; w < 8; ++w)
                table[w] = 0;
        for (uint32_t a = 0; a < (1u << n); ++a)
                if ((v.w[a >> 6] >> (a & 63u)) & 1ull) {
                        table[a >> 5] |= 1u << (a & 31u);
                        nec &= a;
                }
        *nterms    = n;
        *necessary = nec;
        return TRN_OK;
}

// Flat-tree form of a DocumentsOnly step program (k_exec_docs, exec_docs_flat.cuh): every leaf gets a bitmap of its own (slots 0 .. nl-1,
// announced by one [OP_LEAF M_NONE dst = leaf slot] marker each, at the front of the program) that ONE flat (leaf, block) pass over the tile
// fills; the rest of the program becomes slot operations on them, the compiler's own slots moved behind the leaf bitmaps.
// Returns the number of leaves (0: the program stays as it is).
// Leaf bitmaps are numbered by descending block count: the (leaf, block) list of a tile is then ordered from the frequent terms (blocks
// of 1-byte deltas, four codes per decoder step) to the rare ones (2-byte deltas, blocks that straddle the tile), so that the 32 lanes
// of a group mostly walk blocks of the same kind — a rare term's lane among frequent ones kept the whole warp in the loop for its 16-31
// slow steps (those ran at a few of 32 lanes and were as many instructions as the fast ones).
// Afterwards the copies are coalesced (flat_tree_coalesce): `SET d <- s` where s is not read again becomes a renaming of d, so a chain
// like SET t <- leaf; AND t, leaf2; OR acc, t runs in the leaf's own bitmap: fewer operations per tile and — what matters more — fewer
// bitmaps per warp (13 -> 8 for the 8-term trees of the benchmark), i.e. more resident warps.
// rootSlot: in = the compiler's root slot, out = the slot that holds the root docset; slotsInUse: out.
static void     flat_tree_coalesce(std::vector<DevStep> &steps, size_t opsBegin, uint32_t nl, uint32_t &rootSlot, uint32_t &slotsInUse);
static uint32_t flat_tree_transform(std::vector<DevStep> &steps, size_t begin, uint32_t next_slot, const std::vector<DevTerm> &terms, uint32_t &rootSlot,
                                    uint32_t &slotsInUse) {
        uint32_t nl{0};
        for (size_t i = begin; i < steps.size(); ++i)
                nl += steps[i].op == OP_LEAF && steps[i].mode != M_NONE;
        uint32_t nops{nl}; // slot operations of the transformed program: one per decoding leaf + every non-leaf step
        for (size_t i = begin; i < steps.size(); ++i)
                nops += steps[i].op != OP_LEAF;
        if (nl < 2 || nl > 16 || nl + next_slot > 30 || nops > 32)
                return 0; // (the kernel keeps leaves and slot operations in lane registers: <= 16 leaves, <= 32 operations, slots < 32)
        for (size_t i = begin; i < steps.size(); ++i)
                if (steps[i].op == OP_COUNT_GE && steps[i].term > 15u)
                        return 0;
        const std::vector<DevStep> prog(steps.begin() + begin, steps.end());
        steps.resize(begin);
        std::vector<DevStep> leaves;
        for (const auto &st : prog)
                if (st.op == OP_LEAF && st.mode != M_NONE)
                        leaves.push_back(st);
        std::vector<uint32_t> order(nl), slotOf(nl); // order[k]: program leaf held by bitmap k; slotOf: its inverse
        for (uint32_t j = 0; j < nl; ++j)
                order[j] = j;
        auto blocksOf = [&](uint32_t j) { return leaves[j].term == kEmptyTerm ? 0u : terms[leaves[j].term].nblocks; };
        std::stable_sort(order.begin(), order.end(), [&](uint32_t a, uint32_t b) { return blocksOf(a) > blocksOf(b); });
        for (uint32_t k = 0; k < nl; ++k) {
                slotOf[order[k]] = k;
                DevStep L        = leaves[order[k]]; // decode marker: term -> leaf bitmap k
                L.mode           = M_NONE;
                L.dst            = uint8_t(k);
                L.src            = 0;
                L.flags          = 0;
                steps.push_back(L);
        }
        uint32_t li{0};
        for (auto st : prog) {
                if (st.op == OP_LEAF) {
                        if (st.mode == M_NONE)
                                continue; // nothing to do in DocumentsOnly mode
                        DevStep S;
                        std::memset(&S, 0, sizeof(S));
                        S.op    = OP_SLOT;
                        S.mode  = st.mode;
                        S.dst   = uint8_t(st.dst + nl);
                        S.src   = uint8_t(slotOf[li++]);
                        S.flags = st.flags;
                        steps.push_back(S);
                        continue;
                }
                st.dst = uint8_t(st.dst + nl); // compiler slots live behind the leaf bitmaps
                if (st.op == OP_SLOT || st.op == OP_COUNT_ADD || st.op == OP_COUNT_GE)
                        st.src = uint8_t(st.src + nl);
                steps.push_back(st);
        }
        rootSlot += nl;
        slotsInUse = nl + next_slot;
        flat_tree_coalesce(steps, begin + nl, nl, rootSlot, slotsInUse);
        return nl;
}

static void flat_tree_coalesce(std::vector<DevStep> &steps, size_t opsBegin, uint32_t nl, uint32_t &rootSlot, uint32_t &slotsInUse) {
        std::vector<DevStep> ops(steps.begin() + std::ptrdiff_t(opsBegin), steps.end());
        for (const auto &o : ops)
                if (o.op != OP_SLOT && o.op != OP_CLEAR)
                        return; // (counter planes address slot RANGES: left alone)
        auto reads = [](const DevStep &o, uint32_t x) { // does o read slot x?
                if (o.op != OP_SLOT)
                        return false;
                if (o.mode == M_NONE)
                        return o.dst == x; // emptiness test only
                return o.src == x || (o.mode != M_SET && o.dst == x);
        };
        auto overwrites = [](const DevStep &o, uint32_t x) { return o.dst == x && (o.op == OP_CLEAR || (o.op == OP_SLOT && o.mode == M_SET)); };
        // x is dead behind operation i: nothing reads it before it is overwritten, and it is not the root
        auto dead = [&](size_t i, uint32_t x) {
                for (size_t j = i + 1; j < ops.size(); ++j) {
                        if (reads(ops[j], x))
                                return false;
                        if (overwrites(ops[j], x))
                                return true;
                }
                return x != rootSlot;
        };
        // CLEAR d ... OR d, x (nothing touching d in between)  ==  SET d <- x
        std::vector<uint8_t> drop(ops.size(), 0);
        for (size_t i = 0; i < ops.size(); ++i) {
                if (ops[i].op != OP_CLEAR)
                        continue;
                const uint32_t d = ops[i].dst;
                for (size_t j = i + 1; j < ops.size(); ++j) {
                        const bool touches = ops[j].dst == d || (ops[j].op == OP_SLOT && ops[j].src == d);
                        if (!touches)
                                continue;
                        if (ops[j].op == OP_SLOT && ops[j].mode == M_OR && ops[j].dst == d && ops[j].src != d) {
                                ops[j].mode = M_SET;
                                drop[i]     = 1;
                        }
                        break;
                }
        }
        // forward renaming: ren[name] = the physical slot that holds it, holder[slot] = the name it holds (the compiler hands slot numbers
        // out again, so a name that is overwritten must not land in a slot that meanwhile carries another live name)
        uint32_t ren[32], holder[32];
        for (uint32_t i = 0; i < 32; ++i)
                ren[i] = holder[i] = i;
        auto deadFrom = [&](size_t i, uint32_t x) { // like dead(), operation i included
                if (x >= 32u)
                        return true;
                if (i < ops.size() && reads(ops[i], x))
                        return false;
                if (i < ops.size() && overwrites(ops[i], x))
                        return true;
                return dead(i, x);
        };
        std::vector<DevStep> out;
        for (size_t i = 0; i < ops.size(); ++i) {
                if (drop[i])
                        continue;
                DevStep o = ops[i];
                if (o.op == OP_SLOT && o.mode == M_SET && o.src != o.dst && dead(i, o.src)) {
                        const uint32_t p = ren[o.src];
                        if (holder[ren[o.dst]] == o.dst)
                                holder[ren[o.dst]] = 0xffu;
                        ren[o.dst] = p;
                        holder[p]  = o.dst;
                        if (o.flags & F_BREAK_IF_EMPTY) { // the emptiness test stays, on the slot that now carries the name
                                o.mode = M_NONE;
                                o.dst  = uint8_t(p);
                                o.src  = uint8_t(p);
                                out.push_back(o);
                        }
                        continue;
                }
                if (o.op == OP_SLOT)
                        o.src = uint8_t(ren[o.src]);
                if (o.op == OP_CLEAR || (o.op == OP_SLOT && o.mode == M_SET)) { // a full overwrite: the name needs a slot nobody lives in
                        uint32_t p = ren[o.dst];
                        if (holder[p] != o.dst && !deadFrom(i, holder[p])) {
                                p = 0xffu;
                                for (uint32_t k = 0; k < 31u && p == 0xffu; ++k) {
                                        const uint32_t q = k + nl < 31u ? k + nl : k + nl - 31u; // compiler slots first, then leaf bitmaps already consumed
                                        if (deadFrom(i, holder[q]) && !(o.op == OP_SLOT && q == o.src))
                                                p = q;
                                }
                                if (p == 0xffu)
                                        return; // (cannot happen: the program had a slot for every live name) leave the program as it was
                        }
                        ren[o.dst] = p;
                        holder[p]  = o.dst;
                }
                o.dst = uint8_t(ren[o.dst]);
                out.push_back(o);
        }
        rootSlot = ren[rootSlot];
        // compiler slots still in use, renumbered densely behind the leaf bitmaps
        uint32_t map[32];
        uint32_t next = nl;
        for (uint32_t i = 0; i < 32; ++i)
                map[i] = i < nl ? i : 0xffu;
        auto use = [&](uint32_t x) {
                if (x >= nl && map[x] == 0xffu)
                        map[x] = next++;
        };
        for (const auto &o : out) {
                use(o.dst);
                if (o.op == OP_SLOT)
                        use(o.src);
        }
        use(rootSlot);
        for (auto &o : out) {
                o.dst = uint8_t(map[o.dst]);
                if (o.op == OP_SLOT)
                        o.src = uint8_t(map[o.src]);
        }
        rootSlot   = map[rootSlot];
        slotsInUse = next;
        steps.resize(opsBegin);
        steps.insert(steps.end(), out.begin(), out.end());
}

extern "C" int trn_debug_compile(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, const trn_qnode *nodes, uint32_t nnodes,
                                 uint32_t root, int scored, trn_debug_step *out, uint32_t cap, uint32_t *nsteps, uint32_t *root_slot, uint32_t *nslots, char *err,
                                 size_t errcap) {
        static_assert(sizeof(trn_debug_step) == sizeof(DevStep), "trn_debug_step mirrors DevStep");
        auto seterr = [&](const std::string &m, int rc) {
                if (err && errcap) {
                        std::strncpy(err, m.c_str(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                return rc;
        };
        if (!index || !terms || !nodes || !nnodes || !out || !nsteps || !root_slot || !nslots || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || scored < 0 ||
            scored > 2)
                return seterr("bad arguments", TRN_ERR_ARG);
        BlockDirectory dir;
        try {
                build_directory(codec, index, nbytes, terms, nterms, 1, dir);
        } catch (const std::exception &e) {
                return seterr(e.what(), TRN_ERR_FORMAT);
        }
        const std::vector<DevTerm> ht = dev_terms(dir, terms, nterms);
        std::vector<DevStep> steps;
        Compiler             cc(nodes, nnodes, ht, scored == 1, root, steps);
        cc.allow_phrase         = codec == TRN_CODEC_GOOGLE; // as trn_debug_plan: the hits are inline (LUCENE would need its hits.data)
        int                  rs = cc.run();
        if (rs < 0)
                return seterr(cc.err, cc.unsupported ? TRN_ERR_UNSUPPORTED : TRN_ERR_ARG);
        uint32_t treeLeaves{0}, treeSlotsInUse{0};
        if (scored == 2) { // DocumentsOnly program in its flat-tree form (what the second k_exec_docs launch runs)
                uint32_t root2 = uint32_t(rs);
                treeLeaves     = flat_tree_transform(steps, 0, cc.next_slot, ht, root2, treeSlotsInUse);
                if (treeLeaves)
                        rs = int(root2);
        }
        if (steps.size() > cap)
                return seterr("step buffer too small", TRN_ERR_CAPACITY);
        std::memcpy(out, steps.data(), steps.size() * sizeof(DevStep));
        *nsteps    = uint32_t(steps.size());
        *root_slot = uint32_t(rs);
        *nslots    = (treeLeaves ? treeSlotsInUse : cc.next_slot) + 1; // + the scratch slot of the kernels
        return TRN_OK;
}

// =================================================================================================== batch planner
PlanConfig trn::plan_config_from_env() {
        PlanConfig pc;
        if (const char *e = getenv("TRN_CAND_COST"))
                pc.cand_cost = std::max(0, atoi(e));
        if (const char *e = getenv("TRN_DOCS_SHIFT")) {
                const int v = atoi(e);
                if (v >= 13 && v <= 17)
                        pc.docs_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_TREE_SHIFT")) {
                const int v = atoi(e);
                if (v == 0 || (v >= 10 && v <= 14))
                        pc.tree_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_RUN_TILES")) {
                const int v = atoi(e);
                if (v >= 1 && v <= 4096)
                        pc.run_tiles = uint32_t(v);
        }
        if (const char *e = getenv("TRN_FLAT_SCORED"))
                pc.flat_scored = atoi(e) != 0;
        if (const char *e = getenv("TRN_SCORED_SHIFT")) {
                const int v = atoi(e);
                if (v == 13 || v == 14)
                        pc.scored_shift = uint32_t(v);
        }
        if (const char *e = getenv("TRN_DENSE_BITMAPS"))
                pc.dense_bitmaps = atoi(e) != 0;
        if (const char *e = getenv("TRN_DENSE_BUDGET")) {
                const double v = atof(e);
                if (v >= 0.0 && v <= 1.0)
                        pc.dense_budget = v;
        }
        if (const char *e = getenv("TRN_PROBE_BITMAPS"))
                pc.probe_bitmaps = atoi(e) != 0;
        if (const char *e = getenv("TRN_PROBE_RATIO")) {
                const double v = atof(e);
                if (v > 0.0)
                        pc.probe_ratio = v;
        }
        if (const char *e = getenv("TRN_PROBE_BUDGET")) {
                const double v = atof(e);
                if (v >= 0.0)
                        pc.probe_budget = v;
        }
        if (const char *e = getenv("TRN_DENSE_RUNS"))
                pc.dense_runs = atoi(e) != 0;
        if (const char *e = getenv("TRN_MIXED_RUNS"))
                pc.mixed_runs = atoi(e) != 0;
        if (const char *e = getenv("TRN_CAND_RUNS"))
                pc.cand_runs = atoi(e) != 0;
        return pc;
}

trn::GroupStarts trn::group_starts(const BlockDirectory &dir) {
        GroupStarts g;
        g.base.resize(dir.terms.size());
        uint64_t n{0};
        for (size_t t = 0; t < dir.terms.size(); ++t) {
                g.base[t] = uint32_t(n);
                n += (dir.terms[t].nblocks + 31u) / 32u;
        }
        g.first.resize(n);
        for (size_t t = 0; t < dir.terms.size(); ++t) {
                const TermDir &T = dir.terms[t];
                for (uint32_t gr = 0; gr < (T.nblocks + 31u) / 32u; ++gr)
                        g.first[g.base[t] + gr] = gr ? dir.blk_last[T.dir_begin + 32u * gr - 1u] + 1u : T.first_doc;
        }
        return g;
}

void trn::dense_span(const DevTerm &T, uint64_t &base, uint64_t &words) {
        base             = (uint64_t(T.first_doc) >> kDenseAlignShift) << kDenseAlignShift;
        const uint64_t e = ((uint64_t(T.last_doc) >> kDenseAlignShift) + 1) << kDenseAlignShift; // 2^32 for a term in the top tile
        words            = (e - base) >> 5;
}

trn::DenseSelection trn::select_dense_terms(const PlanConfig &cfg, const std::vector<DevTerm> &terms, uint64_t index_bytes) {
        DenseSelection s;
        s.off.assign(terms.size(), kDenseNone);
        if (cfg.codec != TRN_CODEC_GOOGLE || !cfg.dense_bitmaps)
                return s;
        std::vector<uint32_t> cand;
        for (uint32_t t = 0; t < terms.size(); ++t) {
                uint64_t base, words;
                dense_span(terms[t], base, words);
                if (terms[t].nblocks && words * 4 <= terms[t].chunk_len)
                        cand.push_back(t);
        }
        std::stable_sort(cand.begin(), cand.end(), [&](uint32_t a, uint32_t b) { return terms[a].documents > terms[b].documents; });
        const double budget = cfg.dense_budget * double(index_bytes);
        for (uint32_t t : cand) {
                uint64_t base, words;
                dense_span(terms[t], base, words);
                if (double((s.words + words) * 4) > budget)
                        break;
                s.off[t] = uint32_t(s.words);
                s.order.push_back(t);
                s.words += words;
        }
        return s;
}

trn::DenseSelection trn::select_probe_terms(const PlanConfig &cfg, const std::vector<DevTerm> &terms, uint64_t index_bytes, const DenseSelection &dense) {
        DenseSelection s;
        s.off = dense.off;
        if (cfg.codec != TRN_CODEC_GOOGLE || !cfg.dense_bitmaps || !cfg.probe_bitmaps)
                return s;
        std::vector<uint32_t> cand;
        for (uint32_t t = 0; t < terms.size(); ++t) {
                uint64_t base, words;
                dense_span(terms[t], base, words);
                if (terms[t].nblocks && dense.off[t] == kDenseNone && double(words * 4) <= cfg.probe_ratio * double(terms[t].chunk_len))
                        cand.push_back(t);
        }
        std::stable_sort(cand.begin(), cand.end(), [&](uint32_t a, uint32_t b) { return terms[a].documents > terms[b].documents; });
        const double budget = cfg.probe_budget * double(index_bytes);
        for (uint32_t t : cand) {
                uint64_t base, words;
                dense_span(terms[t], base, words);
                if (double((s.words + words) * 4) > budget || dense.words + s.words + words >= (1ull << 32))
                        break;
                s.off[t] = uint32_t(dense.words + s.words);
                s.order.push_back(t);
                s.words += words;
        }
        return s;
}

void trn::build_directory(int codec, const uint8_t *index, uint64_t nbytes, const trn_term *terms, uint32_t nterms, int threads, BlockDirectory &dir) {
        std::vector<term_index_ctx> t(nterms);
        for (uint32_t i = 0; i < nterms; ++i) {
                t[i].documents = terms[i].documents;
                t[i].offset    = terms[i].chunk_off;
                t[i].size      = terms[i].chunk_len;
        }
        build_block_directory(codec == TRN_CODEC_GOOGLE ? Codec::Google : Codec::Lucene, index, nbytes, t.data(), nterms, threads, dir);
}

std::vector<DevTerm> trn::dev_terms(const BlockDirectory &dir, const trn_term *terms, uint32_t nterms) {
        std::vector<DevTerm> ht(nterms);
        for (uint32_t i = 0; i < nterms; ++i) {
                ht[i].documents = dir.terms[i].documents;
                ht[i].dir_begin = dir.terms[i].dir_begin;
                ht[i].nblocks   = dir.terms[i].nblocks;
                ht[i].first_doc = dir.terms[i].first_doc;
                ht[i].last_doc  = dir.terms[i].last_doc;
                ht[i].chunk_len = terms[i].chunk_len;
                ht[i].tf_begin  = dir.terms[i].tf_begin;
                ht[i].tf_base   = dir.terms[i].tf_base;
                ht[i].tf_shift  = dir.terms[i].tf_shift;
        }
        return ht;
}

void trn::docid_span(const std::vector<DevTerm> &terms, uint32_t &min_docid, uint32_t &max_docid) {
        const bool recorded = max_docid != 0;
        min_docid           = 0xffffffffu;
        for (const auto &T : terms)
                if (T.nblocks) {
                        min_docid = std::min(min_docid, T.first_doc);
                        if (!recorded)
                                max_docid = std::max(max_docid, T.last_doc);
                }
}

static int fail(std::string &err, int code, const std::string &m) {
        err = m;
        return code;
}

int trn::plan_batch(const PlanConfig &cfg, const std::vector<DevTerm> &terms, const uint32_t *dense_off, const trn_query *queries, uint32_t nq, int mode,
                    uint32_t k, BatchPlan &out, std::string &err, const uint2 *clip, const GroupStarts *groups) {
        out                = BatchPlan{};
        const bool scored  = mode == TRN_MODE_SCORED_ALL || mode == TRN_MODE_SCORED_TOPK;
        if (mode == TRN_MODE_MATCHED_TERMS) { // the DocumentsOnly program, plus what the collect pass runs per match
                if (!cfg.allow_phrase)
                        return fail(err, TRN_ERR_UNSUPPORTED, "the default exec mode needs the hits: a LUCENE source runs it once its hits.data has been uploaded (trn_upload_hits)");
                if (const int rc = plan_collect(terms, queries, nq, out.collect, err); rc != TRN_OK)
                        return rc;
        }
        const bool google  = cfg.codec == TRN_CODEC_GOOGLE;
        const double width = double(cfg.max_docid) - double(std::min(cfg.min_docid, cfg.max_docid)) + 1.0; // docID span of THIS source
        // docID tile of the step-program launch: set queries run one warp per tile (k_exec_docs) on larger tiles; scored queries keep a
        // CTA-wide fp32 score tile (k_exec_tiles).
        const uint32_t execShift = std::max(scored ? cfg.tile_shift : cfg.docs_shift, cfg.tile_shift);
        out.exec_shift           = execShift;
        auto &steps              = out.steps;
        bool  anyCandidate{false}, anyMembership{false};
        out.queries.assign(nq, DevQuery{});
        for (uint32_t q = 0; q < nq; ++q) {
                const auto &Q = queries[q];
                if (!Q.nodes || !Q.nnodes)
                        return fail(err, TRN_ERR_ARG, "empty query");
                Compiler cc(Q.nodes, Q.nnodes, terms, scored, Q.root, steps);
                cc.allow_phrase = cfg.allow_phrase;
                // the default exec mode makes a GenericDocsSetSpan for every root (exec.cpp:452-505), which honours a root Filter
                cc.reference_quirks = mode != TRN_MODE_MATCHED_TERMS;
                auto &dq        = out.queries[q];
                dq.step_begin   = uint32_t(steps.size());
                const int rs    = cc.run();
                out.any_phrase |= cc.has_phrase;
                if (rs < 0)
                        return fail(err, cc.unsupported ? TRN_ERR_UNSUPPORTED : TRN_ERR_ARG, "query " + std::to_string(q) + ": " + cc.err);
                dq.nsteps    = uint32_t(steps.size()) - dq.step_begin;
                dq.root_slot = uint32_t(rs);
                // conjunction / disjunction whose operands are all terms (matchallterms / matchanyterms runs): TRN_ROUTE_FLAT_AND / _OR
                uint32_t flatList{TRN_ROUTE_STEPS};
                {
                        const auto &R = Q.nodes[cc.root];
                        if ((R.kind == TRN_NODE_AND || R.kind == TRN_NODE_OR) && R.nchildren <= 16) {
                                bool allTerms{true};
                                for (uint32_t ch = 0; ch < R.nchildren; ++ch)
                                        allTerms &= Q.nodes[R.first_child + ch].kind == TRN_NODE_TERM;
                                if (allTerms) {
                                        flatList = R.kind == TRN_NODE_AND ? TRN_ROUTE_FLAT_AND : TRN_ROUTE_FLAT_OR;
                                        // one bitmap per operand.  This also raises the slot count where the plan does not run as a flat AND
                                        // (LUCENE, scored, candidate-driven), which does not need the slots: left as it is (the slot count sets the
                                        // launch's occupancy, so changing it is a tuning change).
                                        if (R.kind == TRN_NODE_AND && R.nchildren <= 3)
                                                out.nslots = std::max<uint32_t>(out.nslots, R.nchildren);
                                }
                        }
                }
                out.postings += cc.postings;
                out.bytes += cc.bytes;
                Range r = cc.range(cc.root); // cc.root: the effective root (see apply_reference_root_filter_quirk)
                if (clip) { // no match lies outside the query's allow set: its tiles there are not evaluated
                        r.lo = std::max(r.lo, clip[q].x);
                        r.hi = std::min(r.hi, clip[q].y);
                }
                // Flat scored disjunction (a k-term OR / a single term, every leaf scoring with a weight >= +0.0) on the LUCENE codec:
                // k_score_flat (score_flat.cuh) instead of the step program
                bool flatScored{false};
                if (scored && cfg.flat_scored && !google && execShift >= 13) {
                        const auto &R = Q.nodes[cc.root];
                        uint32_t    f0{cc.root}, nl{1};
                        bool        ok = R.kind == TRN_NODE_TERM;
                        if (R.kind == TRN_NODE_OR && R.nchildren <= cfg.score_flat_max_leaves) {
                                ok = true;
                                f0 = R.first_child;
                                nl = R.nchildren;
                                for (uint32_t ch = 0; ch < nl; ++ch)
                                        ok &= Q.nodes[f0 + ch].kind == TRN_NODE_TERM;
                        }
                        for (uint32_t ch = 0; ok && ch < nl; ++ch) {
                                const double w = Q.nodes[f0 + ch].weight;
                                ok             = std::isfinite(w) && !std::signbit(w); // the -0.0f "untouched" sentinel of the score tile needs contributions >= +0.0
                        }
                        if (ok) {
                                flatScored = true;
                                steps.resize(dq.step_begin); // no step program
                                dq.nsteps = 0;
                                FlatQuery fq;
                                std::memset(&fq, 0, sizeof(fq));
                                fq.qid        = q;
                                fq.leaf_begin = uint32_t(out.leaves.size());
                                fq.nleaf      = nl;
                                for (uint32_t ch = 0; ch < nl; ++ch) {
                                        FlatLeaf L;
                                        L.term = Q.nodes[f0 + ch].term;
                                        L.pad  = 0;
                                        L.idf  = Q.nodes[f0 + ch].weight;
                                        out.leaves.push_back(L);
                                }
                                out.flat.push_back(fq);
                        }
                }
                const uint32_t planSlots = cc.next_slot + 1; // + scratch slot (applied below, once the path of the query is known)
                // Candidate-driven evaluation (exec_docs_cand.cuh) when some term that EVERY match must hold is sparse: cost follows that
                // lead's postings (~cand_cost/2 warp-instructions per 32 candidates and probed term; the crossover was tuned on the and2
                // workload: 900 beats 450 and 1500) instead of the docID space (~1500 per tile + ~27 per block in it).
                // The boolean function of the tree over its (<= 8 distinct) terms is tabulated here; the device probes every term for
                // each candidate and looks the membership bits up.
                bool candidate{false};
                if (!scored && google && cfg.cand_cost > 0 && !r.empty() && !cc.has_phrase) {
                        uint32_t tv[8], n{0}; // distinct non-empty terms below the effective root
                        if (distinct_terms(Q.nodes, Q.nnodes, cc.root, &terms, tv, n) == TRN_OK && n >= 2) {
                                // truth vectors: bit `bits` of vec(node) = value of the node under the term assignment `bits` (bit j = tv[j])
                                uint8_t  truth[256];
                                uint32_t necessary{(1u << n) - 1u};
                                bool     any{false};
                                if (flatList == TRN_ROUTE_FLAT_AND && n == Q.nodes[cc.root].nchildren) { // all-term conjunction: only the all-ones assignment matches
                                        std::memset(truth, 0, sizeof(truth));
                                        truth[(1u << n) - 1u] = 1;
                                        any                   = true;
                                } else {
                                        const TruthVec tvec = truth_vector(Q.nodes, cc.root, tv, n);
                                        for (uint32_t bits = 0; bits < (1u << n); ++bits) {
                                                truth[bits] = uint8_t((tvec.w[bits >> 6] >> (bits & 63u)) & 1ull);
                                                if (truth[bits]) {
                                                        necessary &= bits;
                                                        any = true;
                                                }
                                        }
                                }
                                if (any && necessary) {
                                        // probe order: the lead (rarest necessary term), the other necessary terms rarest first (they filter),
                                        // then the rest
                                        uint32_t order[8], nn{0}, no{0};
                                        for (uint32_t j = 0; j < n; ++j)
                                                if ((necessary >> j) & 1u)
                                                        order[no++] = j;
                                        nn = no;
                                        for (uint32_t j = 0; j < n; ++j)
                                                if (!((necessary >> j) & 1u))
                                                        order[no++] = j;
                                        auto byBlocks = [&](uint32_t x, uint32_t y) { return terms[tv[x]].nblocks < terms[tv[y]].nblocks; };
                                        std::sort(order, order + nn, byBlocks);
                                        std::sort(order + nn, order + n, byBlocks);
                                        const uint32_t lead = tv[order[0]];
                                        double         blocks{0};
                                        for (uint32_t j = 0; j < n; ++j)
                                                blocks += terms[tv[j]].nblocks;
                                        const bool   flatAnd = flatList == TRN_ROUTE_FLAT_AND;
                                        const double perTile = double(1ull << execShift) / width;
                                        const double lhs     = double(n - 1) * terms[lead].nblocks * perTile * double(cfg.cand_cost);
                                        const double rhs     = 1500.0 + (flatAnd ? 0.0 : 150.0 * n) + blocks * perTile * (flatAnd ? 27.0 : 35.0);
                                        if (lhs < rhs) {
                                                // replace the step program: terms in probe order, then the truth table re-indexed to probe positions
                                                steps.resize(dq.step_begin);
                                                for (uint32_t j = 0; j < n; ++j)
                                                        cc.push(OP_LEAF, M_NONE, 0, 0, 0, tv[order[j]], 0.0);
                                                uint32_t words[8] = {0, 0, 0, 0, 0, 0, 0, 0};
                                                for (uint32_t pb = 0; pb < (1u << n); ++pb) { // pb: bit j = term at probe position j
                                                        uint32_t bits{0};
                                                        for (uint32_t j = 0; j < n; ++j)
                                                                if ((pb >> j) & 1u)
                                                                        bits |= 1u << order[j];
                                                        if (truth[bits])
                                                                words[pb >> 5] |= 1u << (pb & 31u);
                                                }
                                                for (uint32_t w = 0; w < 8; w += 4) {
                                                        DevStep st;
                                                        std::memset(&st, 0, sizeof(st));
                                                        st.op   = OP_TABLE;
                                                        st.dst  = uint8_t(w);
                                                        st.term = words[w];
                                                        st.pad2 = words[w + 1];
                                                        uint64_t hi = uint64_t(words[w + 2]) | (uint64_t(words[w + 3]) << 32);
                                                        std::memcpy(&st.idf, &hi, 8);
                                                        steps.push_back(st);
                                                }
                                                dq.nsteps    = uint32_t(steps.size()) - dq.step_begin;
                                                dq.root_slot = nn;
                                                candidate    = true;
                                                dq.tile_lo   = 0;
                                                dq.ntiles    = (terms[lead].nblocks + 31u) / 32u;
                                                anyCandidate = true;
                                                anyMembership |= nn < n;
                                        }
                                }
                        }
                }
                // Flat-tree path (exec_docs_flat.cuh): a DocumentsOnly tree that is neither an all-term run nor candidate-driven decodes ALL its
                // leaves of a tile in one flat (leaf, block) pass — each leaf into a bitmap of its own — and then runs slot operations only.
                // The per-leaf groups of the step-program path ran at a third of the lanes with up to 8 live bitmaps per warp; here
                // the lanes are packed across leaves, and a smaller tile pays for the extra bitmaps.
                bool treeFlat{false};
                if (!scored && !candidate && flatList == TRN_ROUTE_STEPS && google && cfg.tree_shift && !r.empty() && !cc.has_phrase) {
                        uint32_t       root2 = dq.root_slot, inUse{0};
                        const uint32_t nl    = flat_tree_transform(steps, dq.step_begin, cc.next_slot, terms, root2, inUse);
                        if (nl) {
                                dq.nsteps      = uint32_t(steps.size()) - dq.step_begin;
                                dq.root_slot   = root2;
                                out.tree_slots = std::max(out.tree_slots, inUse);
                                treeFlat       = true;
                        }
                }
                if (!flatScored && !treeFlat)
                        out.nslots = std::max(out.nslots, planSlots);
                // the path this query takes.  The LUCENE instantiation of k_exec_docs has no flat AND / OR form: it runs those plans as step
                // programs.
                if (scored)
                        dq.route = flatScored ? TRN_ROUTE_SCORE_FLAT : TRN_ROUTE_EXEC_TILES;
                else
                        dq.route = candidate ? TRN_ROUTE_CANDIDATE : treeFlat ? TRN_ROUTE_FLAT_TREE : google ? flatList : TRN_ROUTE_STEPS;
                const uint32_t qshift = flatScored ? cfg.scored_shift : (treeFlat ? cfg.tree_shift : execShift); // per-path tile
                if (candidate) {
                } else if (r.empty()) {
                        dq.tile_lo = 0;
                        dq.ntiles  = 0;
                } else {
                        dq.tile_lo = r.lo >> qshift;
                        dq.ntiles  = (r.hi >> qshift) - dq.tile_lo + 1;
                }
                dq.item_base = uint32_t(out.items);
                dq.gen_base  = uint32_t(out.gen_items);
                dq.gen_base2 = uint32_t(out.gen_items2);
                out.items += dq.ntiles;
                if (treeFlat)
                        out.gen_items2 += dq.ntiles;
                else if (!flatScored)
                        out.gen_items += dq.ntiles;
                if (out.items >= (1ull << 32))
                        return fail(err, TRN_ERR_CAPACITY, "batch has more than 2^32 (query, tile) work items; split it");
                const uint64_t rangeDocs = r.empty() ? 0 : uint64_t(r.hi) - r.lo + 1;
                uint64_t       segWords  = std::min(cc.bound(cc.root), rangeDocs);
                // compact results (planned as DocumentsOnly): a tile wider than 2^16 docIDs has no offset form (exec_docs.cuh
                // tile_encoding), so every tile that holds a match takes its bitmap, 2^qshift / 32 words however few documents it holds.
                // (Sized by the docID count alone, a batch of sparse phrase queries at TRN_DOCS_SHIFT=17 overflowed its segment buffer.)
                if (!candidate && qshift > 16u)
                        segWords = std::max(segWords, std::min<uint64_t>(segWords, dq.ntiles) << (qshift - 5u));
                out.seg_cap += segWords;
                dq.cand_base = uint32_t(out.cand_total);
                dq.cand_cap  = uint32_t(std::min<uint64_t>(uint64_t(dq.ntiles) * k, 0xffffffffull));
                if (flatScored) {
                        auto &fq      = out.flat.back();
                        fq.tile_lo    = dq.tile_lo;
                        fq.ntiles     = dq.ntiles;
                        fq.nruns      = (dq.ntiles + cfg.run_tiles - 1u) / cfg.run_tiles;
                        fq.item_base  = dq.item_base;
                        fq.local_base = uint32_t(out.flat_items);
                        out.flat_items += dq.ntiles;
                        out.max_runs = std::max(out.max_runs, fq.nruns);
                        dq.cand_cap  = uint32_t(std::min<uint64_t>(uint64_t(fq.nruns) * k, 0xffffffffull));
                        fq.cand_base = dq.cand_base;
                        fq.cand_cap  = dq.cand_cap;
                }
                if (mode == TRN_MODE_SCORED_TOPK) {
                        out.cand_total += dq.cand_cap;
                        if (out.cand_total >= (1ull << 32))
                                return fail(err, TRN_ERR_CAPACITY, "top-k candidate space exceeds 2^32 entries; split the batch");
                }
        }
        if (uint64_t(out.max_runs) * out.flat.size() >= (1ull << 32))
                return fail(err, TRN_ERR_CAPACITY, "batch has more than 2^32 (run, query) work items; split it");
        if (anyCandidate) { // the candidate array + one gather buffer must fit a warp's share of shared memory
                const uint32_t slotBytes = (1u << execShift) / 8u, stageB = cfg.docs_stage_bytes, need = cfg.cand_smem_bytes[anyMembership];
                if (need > stageB)
                        out.nslots = std::max(out.nslots, (need - stageB + slotBytes - 1u) / slotBytes);
        }
        // a flat conjunction keeps one bitmap per operand: with more operands than the launch has slots (final only here) it runs as a
        // step program.  One whose operands all have a resident bitmap decodes nothing: it joins the run-major ticket space (dense_runs) —
        // except beside a phrase plan, whose instantiation of k_exec_docs does not carry that path.
        const bool runs = dense_off && cfg.dense_runs && google && !scored && !out.any_phrase;
        // A flat AND with exactly one operand without a bitmap decodes that operand (the lead) once per run and probes the others' bitmaps
        // per candidate (exec_docs.cuh mixed_run_exec) — when the warp's share of shared memory holds the path's candidate array.
        const bool mixedRuns = dense_off && cfg.mixed_runs && google && !scored && !out.any_phrase &&
                               out.nslots * ((1u << execShift) / 8u) + cfg.docs_stage_bytes >= cfg.mixed_smem_bytes;
        std::vector<uint32_t> group, mixed; // the queries of dense_runs, of mixed_runs
        for (uint32_t q = 0; q < nq; ++q) {
                auto &dq = out.queries[q];
                if (dq.route == TRN_ROUTE_FLAT_AND) {
                        uint32_t nleaf{0}, ndecoded{0};
                        bool     known{dq.ntiles != 0};
                        for (uint32_t si = 0; si < dq.nsteps; ++si) {
                                const DevStep &st = steps[dq.step_begin + si];
                                if (st.op == OP_LEAF) {
                                        ++nleaf;
                                        known = known && st.term != kEmptyTerm;
                                        ndecoded += (!dense_off || st.term == kEmptyTerm || dense_off[st.term] == kDenseNone) ? 1u : 0u;
                                }
                        }
                        if (nleaf > out.nslots)
                                dq.route = TRN_ROUTE_STEPS;
                        else if (runs && known && ndecoded == 0)
                                group.push_back(q);
                        else if (mixedRuns && known && ndecoded == 1 && nleaf >= 2 && nleaf <= 32)
                                mixed.push_back(q);
                }
        }
        // (run, query) pairs, counting-sorted by run (queries ascending within a run).  Every tile of such a query lies inside every
        // bitmap operand's span (the query's range is the intersection of the operands' ranges), and so does the run that holds it.
        const uint32_t rs          = kDenseAlignShift - execShift;
        auto           run_tickets = [&](const std::vector<uint32_t> &qs, std::vector<uint2> &tickets) {
                if (qs.empty())
                        return;
                uint32_t r0{0xffffffffu}, r1{0};
                for (uint32_t q : qs) {
                        const auto &dq = out.queries[q];
                        r0             = std::min(r0, dq.tile_lo >> rs);
                        r1             = std::max(r1, (dq.tile_lo + dq.ntiles - 1u) >> rs);
                }
                std::vector<uint32_t> at(size_t(r1 - r0) + 2, 0);
                for (uint32_t q : qs) {
                        const auto &dq = out.queries[q];
                        for (uint32_t r = dq.tile_lo >> rs; r <= (dq.tile_lo + dq.ntiles - 1u) >> rs; ++r)
                                ++at[r - r0 + 1];
                }
                for (size_t i = 1; i < at.size(); ++i)
                        at[i] += at[i - 1];
                tickets.resize(at.back());
                for (uint32_t q : qs) {
                        const auto &dq = out.queries[q];
                        for (uint32_t r = dq.tile_lo >> rs; r <= (dq.tile_lo + dq.ntiles - 1u) >> rs; ++r)
                                tickets[at[r - r0]++] = uint2{q, std::max(dq.tile_lo, r << rs)};
                }
        };
        run_tickets(group, out.dense_runs);
        run_tickets(mixed, out.mixed_runs);
        // Candidate-driven groups, same conditions: {query, group} tickets counting-sorted by the run of the group's first docID (queries
        // ascending within a run, then groups ascending).  The warps in flight then hold neighbouring docID windows of every lead, so
        // the bitmap words and directory entries their probes read are shared through L2 instead of each coming from HBM.
        const bool candRuns = groups && cfg.cand_runs && google && !scored && !out.any_phrase && anyCandidate;
        if (candRuns) {
                constexpr uint32_t    kRuns = 1u << (32 - kDenseAlignShift);
                std::vector<uint32_t> at(kRuns + 1, 0);
                auto                  lead_groups = [&](const DevQuery &dq) { return groups->first.data() + groups->base[steps[dq.step_begin].term]; };
                for (uint32_t q = 0; q < nq; ++q) {
                        const auto &dq = out.queries[q];
                        if (dq.route != TRN_ROUTE_CANDIDATE)
                                continue;
                        const uint32_t *gf = lead_groups(dq);
                        for (uint32_t gr = 0; gr < dq.ntiles; ++gr)
                                ++at[(gf[gr] >> kDenseAlignShift) + 1];
                }
                for (uint32_t i = 1; i <= kRuns; ++i)
                        at[i] += at[i - 1];
                out.cand_runs.resize(at[kRuns]);
                for (uint32_t q = 0; q < nq; ++q) {
                        const auto &dq = out.queries[q];
                        if (dq.route != TRN_ROUTE_CANDIDATE)
                                continue;
                        const uint32_t *gf = lead_groups(dq);
                        for (uint32_t gr = 0; gr < dq.ntiles; ++gr)
                                out.cand_runs[at[gf[gr] >> kDenseAlignShift]++] = uint2{q, gr};
                }
        }
        if (!group.empty() || !mixed.empty() || candRuns) {
                // the step-program launch's own tickets without them (the items keep their item_base)
                out.gen_items = 0;
                for (uint32_t q = 0, g = 0, m = 0; q < nq; ++q) {
                        auto &dq    = out.queries[q];
                        dq.gen_base = uint32_t(out.gen_items);
                        if (g < group.size() && group[g] == q)
                                ++g;
                        else if (m < mixed.size() && mixed[m] == q)
                                ++m;
                        else if (dq.route != TRN_ROUTE_FLAT_TREE)
                                out.gen_items += dq.ntiles;
                }
        }
        // the candidate groups' tickets run the groups' own step-program tickets (gen_base + group), which the launch then skips
        if (candRuns) {
                if (out.gen_items >= (1ull << 31)) { // (the kernel marks a run ticket in bit 31 of its ticket number)
                        out.cand_runs.clear();
                        return TRN_OK;
                }
                out.cand_order.resize(out.cand_runs.size());
                for (size_t i = 0; i < out.cand_runs.size(); ++i)
                        out.cand_order[i] = out.queries[out.cand_runs[i].x].gen_base + out.cand_runs[i].y;
        }
        return TRN_OK;
}

// The collect program of a query (the default exec mode, collect.cuh): its distinct terms, ascending, and its nodes in post order with
// queryexec_ctx::collect_doc_matching_terms' rules (queryexec_ctx.cpp:382-648) — a TERM reports itself, an AND all its children, an OR /
// SOME the children that hold the document, a NOT its required side, an OPTIONAL its main and its opt where opt holds the document, a
// PHRASE all its terms.  A term the source does not hold never holds a document; so does a phrase with such a term.
int trn::plan_collect(const std::vector<DevTerm> &terms, const trn_query *queries, uint32_t nq, CollectPlan &out, std::string &err) {
        out = CollectPlan{};
        out.queries.resize(nq);
        for (uint32_t q = 0; q < nq; ++q) {
                const auto &Q = queries[q];
                const auto *n = Q.nodes;
                if (!n || !Q.nnodes || Q.root >= Q.nnodes || !plan_depth_ok(n, Q.nnodes))
                        return fail(err, TRN_ERR_ARG, "query " + std::to_string(q) + ": bad plan");
                auto held = [&](uint32_t t) { return t != kEmptyTerm && t < terms.size() && terms[t].documents != 0; };
                // the distinct terms below the root
                std::vector<uint32_t> tv, todo{Q.root};
                while (!todo.empty()) {
                        const uint32_t i = todo.back();
                        todo.pop_back();
                        if (n[i].kind == TRN_NODE_TERM) {
                                if (held(n[i].term))
                                        tv.push_back(n[i].term);
                        } else
                                for (uint32_t c = 0; c < n[i].nchildren; ++c)
                                        if (uint32_t(n[i].first_child) + c < Q.nnodes && n[i].first_child > i)
                                                todo.push_back(n[i].first_child + c);
                }
                std::sort(tv.begin(), tv.end());
                tv.erase(std::unique(tv.begin(), tv.end()), tv.end());
                if (tv.size() > kCollectMaxTerms)
                        return fail(err, TRN_ERR_UNSUPPORTED,
                                    "query " + std::to_string(q) + ": the default exec mode takes at most 32 distinct terms per query (" + std::to_string(tv.size()) + ")");
                auto bit = [&](uint32_t t) { return held(t) ? uint32_t(std::lower_bound(tv.begin(), tv.end(), t) - tv.begin()) : kEmptyTerm; };
                auto &cq        = out.queries[q];
                cq.term_begin   = uint32_t(out.terms.size());
                cq.nterms       = uint32_t(tv.size());
                cq.phrase_begin = uint32_t(out.phrases.size());
                cq.prog_begin   = uint32_t(out.prog.size());
                out.terms.insert(out.terms.end(), tv.begin(), tv.end());
                uint32_t    sp{0}, nph{0};
                std::string perr;
                // post order, iteratively (trees are up to 64 levels deep): a node is emitted once all its children have been
                std::vector<std::pair<uint32_t, uint32_t>> st{{Q.root, 0}};
                while (!st.empty() && perr.empty()) {
                        auto [i, c]   = st.back();
                        const auto &X = n[i];
                        CollectOp   o{};
                        if (X.kind == TRN_NODE_TERM || X.kind == TRN_NODE_PHRASE) {
                                st.pop_back();
                                o.kind = CO_TERM;
                                o.arg  = X.kind == TRN_NODE_TERM ? bit(X.term) : kEmptyTerm;
                                if (X.kind == TRN_NODE_PHRASE) {
                                        bool     all{X.nchildren >= 2 && X.nchildren <= 16 && X.first_child > i && uint32_t(X.first_child) + X.nchildren <= Q.nnodes};
                                        uint32_t mask{0};
                                        for (uint32_t k = 0; all && k < X.nchildren; ++k) {
                                                const auto &C = n[X.first_child + k];
                                                all           = C.kind == TRN_NODE_TERM && held(C.term);
                                                if (all)
                                                        mask |= 1u << bit(C.term);
                                        }
                                        if (all) { // (a phrase with a term the source does not hold matches nothing: it stays a TERM that never holds)
                                                if (nph == kCollectMaxPhrases) {
                                                        perr = "the default exec mode takes at most 32 phrase nodes per query";
                                                        break;
                                                }
                                                CollectPhrase F{};
                                                F.arg_begin = uint32_t(out.args.size());
                                                F.k         = X.nchildren;
                                                F.mask      = mask;
                                                for (uint32_t j = 0; j < X.nchildren; j += 4) { // four term ids per OP_ARG step (phrase.cuh phrase_arg)
                                                        auto   t = [&](uint32_t k) { return k < X.nchildren ? n[X.first_child + k].term : 0u; };
                                                        DevStep a;
                                                        std::memset(&a, 0, sizeof(a));
                                                        a.op                = OP_ARG;
                                                        a.term              = t(j);
                                                        a.pad2              = t(j + 1);
                                                        const uint64_t hi   = uint64_t(t(j + 2)) | (uint64_t(t(j + 3)) << 32);
                                                        std::memcpy(&a.idf, &hi, 8);
                                                        out.args.push_back(a);
                                                }
                                                out.phrases.push_back(F);
                                                o.kind = CO_PHRASE;
                                                o.arg  = nph++;
                                        }
                                }
                        } else if (c < X.nchildren) {
                                if (X.first_child <= i || uint32_t(X.first_child) + X.nchildren > Q.nnodes) {
                                        perr = "children must follow their parent in the node array";
                                        break;
                                }
                                st.back().second = c + 1;
                                st.push_back({uint32_t(X.first_child) + c, 0});
                                continue;
                        } else {
                                st.pop_back();
                                if ((X.kind == TRN_NODE_NOT || X.kind == TRN_NODE_OPTIONAL) && X.nchildren != 2) {
                                        perr = "NOT and OPTIONAL nodes have two children";
                                        break;
                                }
                                o.kind      = X.kind == TRN_NODE_AND ? CO_AND : X.kind == TRN_NODE_OR ? CO_OR : X.kind == TRN_NODE_NOT ? CO_NOT : X.kind == TRN_NODE_OPTIONAL ? CO_OPTIONAL : CO_SOME;
                                o.nchildren = X.nchildren;
                                o.min       = uint16_t(X.kind == TRN_NODE_SOME ? std::min<uint32_t>(X.term, 0xffffu) : 0u);
                                o.arg       = 0;
                                sp -= X.nchildren;
                        }
                        out.prog.push_back(o);
                        if (++sp > kCollectMaxStack) {
                                perr = "the query's collect program needs more than 32 pending operands";
                                break;
                        }
                }
                if (!perr.empty())
                        return fail(err, TRN_ERR_UNSUPPORTED, "query " + std::to_string(q) + ": " + perr);
                cq.nphrases = nph;
                cq.nprog    = uint32_t(out.prog.size()) - cq.prog_begin;
        }
        return TRN_OK;
}
