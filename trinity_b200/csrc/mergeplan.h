// The host half of trn_merge_sources: MergeCandidatesCollection::commit() and the term loop of merge() (merge.cpp:6-35, 127-158, 166-395)
// restated as a pure function over the sources' names and tuples.  It reads no postings.  Exported as trn_debug_merge_plan.
//   * candidates: the sources by generation, newest first; two equal generations are refused (merge() EXPECTs them strictly descending)
//   * registries: candidate j masks d iff a NEWER candidate lists d in its updated documents.  Kept as one sorted array of the distinct
//     updated docIDs with the newest candidate that lists each (upd_first): d is masked for j iff upd_first(d) < j — one sort, O(updates)
//   * output terms: a merge of the name lists by terms_cmp (common.h:48: bytewise, a prefix first); holders in candidate order
//   * routes (merge.cpp:166-395): one holder -> append (same codec, empty registry, optimisations on; 0 documents: skip) or re-encode
//     through the decode loop (0 documents: skip); several holders -> IndexSession::merge (all of out_codec, optimisations on) or the
//     generic loop, both over the holders with documents (none: skip).  Only the two decode loops add to sumTermsDocs / sumTermHits.
//   * the GOOGLE skiplist countdown belongs to the one output encoder (google_codec.h:57): appended chunks leave it alone, so the
//     re-encoded terms run it from a fresh encoder's phase, 0.
#pragma once
#include "../../include/trinity_b200.h"
#include <algorithm>
#include <cstdint>
#include <cstring>
#include <string>
#include <vector>

namespace trn {

enum : uint8_t { MERGE_APPEND = 0, MERGE_REENCODE = 1 };

struct MergePart {
        uint32_t cand, term; // candidate (newest first), term index in that candidate's source
};
struct MergeOut {
        uint8_t  route, stats;
        uint32_t part_begin; // parts[part_begin .. next term's part_begin)
};
struct MergePlan {
        std::vector<uint32_t>  order; // order[j] = source of candidate j
        std::vector<MergeOut>  out;   // + a sentinel entry whose part_begin = parts.size()
        std::vector<MergePart> parts;
        std::vector<uint32_t>  upd_docid, upd_first;
        uint32_t               countdown_phase{0};
        bool                   masks(uint32_t cand, uint32_t d) const {
                const auto it = std::lower_bound(upd_docid.begin(), upd_docid.end(), d);
                return it != upd_docid.end() && *it == d && upd_first[size_t(it - upd_docid.begin())] < cand;
        }
};

// terms_cmp (common.h:48): bytewise, on a common prefix the shorter first
inline int merge_terms_cmp(const char *a, size_t la, const char *b, size_t lb) {
        const int r = std::memcmp(a, b, std::min(la, lb));
        return r ? r : (la < lb ? -1 : la > lb ? 1 : 0);
}

// 0 or a TRN_ERR_* with err naming the source and term
inline int plan_merge(int out_codec, const trn_merge_source *src, uint32_t n, bool disable_optimizations, MergePlan &P, std::string &err) {
        P = MergePlan{};
        if ((out_codec != TRN_CODEC_GOOGLE && out_codec != TRN_CODEC_LUCENE) || (n && !src)) {
                err = "trn_merge_sources: bad arguments";
                return TRN_ERR_ARG;
        }
        if (n > TRN_MERGE_MAX_SOURCES) {
                err = "trn_merge_sources: " + std::to_string(n) + " sources: at most 128 (the reference's decoder array, merge.cpp:310-312)";
                return TRN_ERR_ARG;
        }
        std::vector<size_t> len;
        for (uint32_t s = 0; s < n; ++s) {
                const auto &S   = src[s];
                const auto  who = "trn_merge_sources: source " + std::to_string(s) + " (generation " + std::to_string(S.generation) + ")";
                if ((S.codec != TRN_CODEC_GOOGLE && S.codec != TRN_CODEC_LUCENE) || (S.nterms && (!S.terms || !S.names)) || (S.index_bytes && !S.index) ||
                    (S.nupdated && !S.updated_docids)) {
                        err = who + ": bad arguments";
                        return TRN_ERR_ARG;
                }
                if (S.codec == TRN_CODEC_LUCENE && !S.hits && S.nterms) {
                        err = who + ": a LUCENE source needs its hits.data";
                        return TRN_ERR_ARG;
                }
                for (uint32_t t = 0; t < S.nterms; ++t) {
                        const char  *nm = S.names[t];
                        const size_t l  = nm ? std::strlen(nm) : 0;
                        if (!l || l > 64) {
                                err = who + ": term " + std::to_string(t) + ": names are 1 to 64 bytes (Limits::MaxTermLength)";
                                return TRN_ERR_ARG;
                        }
                        if (t && merge_terms_cmp(S.names[t - 1], std::strlen(S.names[t - 1]), nm, l) >= 0) {
                                err = who + ": term " + std::to_string(t) + " [" + nm + "]: names must be strictly ascending in terms_cmp order";
                                return TRN_ERR_ARG;
                        }
                        if (uint64_t(S.terms[t].chunk_off) + S.terms[t].chunk_len > S.index_bytes) {
                                err = who + ": term [" + std::string(nm) + "]: its chunk lies outside the source's index";
                                return TRN_ERR_ARG;
                        }
                }
        }
        P.order.resize(n);
        for (uint32_t s = 0; s < n; ++s)
                P.order[s] = s;
        std::stable_sort(P.order.begin(), P.order.end(), [&](uint32_t a, uint32_t b) { return src[a].generation > src[b].generation; });
        for (uint32_t j = 1; j < n; ++j)
                if (src[P.order[j]].generation == src[P.order[j - 1]].generation) {
                        err = "trn_merge_sources: sources " + std::to_string(P.order[j - 1]) + " and " + std::to_string(P.order[j]) + " share generation " +
                              std::to_string(src[P.order[j]].generation);
                        return TRN_ERR_ARG;
                }
        // registries: (docID, newest candidate listing it)
        {
                std::vector<uint64_t> u;
                for (uint32_t j = 0; j < n; ++j) {
                        const auto &S = src[P.order[j]];
                        for (uint64_t i = 0; i < S.nupdated; ++i)
                                u.push_back((uint64_t(S.updated_docids[i]) << 32) | j);
                }
                std::sort(u.begin(), u.end());
                for (const uint64_t x : u)
                        if (P.upd_docid.empty() || P.upd_docid.back() != uint32_t(x >> 32)) {
                                P.upd_docid.push_back(uint32_t(x >> 32));
                                P.upd_first.push_back(uint32_t(x));
                        }
        }
        // a candidate's registry is empty iff no newer candidate updates a document
        std::vector<uint32_t> first_updater_before(n + 1, 0); // number of candidates < j with updates
        for (uint32_t j = 0; j < n; ++j)
                first_updater_before[j + 1] = first_updater_before[j] + (src[P.order[j]].nupdated ? 1u : 0u);
        // the term merge: k-way over the candidates' sorted name lists
        std::vector<uint32_t> cur(n, 0);
        std::vector<uint32_t> holders;
        holders.reserve(n);
        for (;;) {
                holders.clear();
                const char *best{nullptr};
                size_t      bl{0};
                for (uint32_t j = 0; j < n; ++j) {
                        const auto &S = src[P.order[j]];
                        if (cur[j] == S.nterms)
                                continue;
                        const char  *nm = S.names[cur[j]];
                        const size_t l  = std::strlen(nm);
                        const int    r  = best ? merge_terms_cmp(nm, l, best, bl) : -1;
                        if (r < 0) {
                                holders.clear();
                                best = nm;
                                bl   = l;
                        }
                        if (r <= 0)
                                holders.push_back(j);
                }
                if (holders.empty())
                        break;
                const auto docs = [&](uint32_t j) { return src[P.order[j]].terms[cur[j]].documents; };
                const auto add  = [&](uint8_t route, uint8_t stats, bool only_with_docs) {
                        const uint32_t b = uint32_t(P.parts.size());
                        for (const uint32_t j : holders)
                                if (!only_with_docs || docs(j))
                                        P.parts.push_back({j, cur[j]});
                        if (P.parts.size() > b)
                                P.out.push_back({route, stats, b});
                };
                if (holders.size() == 1) {
                        const uint32_t j = holders[0];
                        if (src[P.order[j]].codec == out_codec && !first_updater_before[j] && !disable_optimizations)
                                add(MERGE_APPEND, 0, true);
                        else
                                add(MERGE_REENCODE, 1, true);
                } else {
                        bool same = true;
                        for (const uint32_t j : holders)
                                same &= src[P.order[j]].codec == out_codec;
                        add(MERGE_REENCODE, same && !disable_optimizations ? 0 : 1, true);
                }
                for (const uint32_t j : holders)
                        ++cur[j];
        }
        P.out.push_back({0, 0, uint32_t(P.parts.size())});
        return TRN_OK;
}

} // namespace trn
