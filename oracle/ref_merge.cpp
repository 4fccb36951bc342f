// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's segment merge (merge.h, merge.cpp), built by oracle/build_merge.sh into
// oracle/_ref/libtrinity_ref_merge.so against the reference objects of libtrinity_ref.so (which holds merge.cpp, segment_index_source.cpp,
// terms.cpp, indexer.cpp and both codecs).
//   * tref_merge opens every source directory as the reference's own SegmentIndexSource, makes a merge_candidate of each (generation, terms
//     view, access proxy, updated documents), commit()s the collection and merge()s it into a fresh GOOGLE or LUCENE IndexSession with the
//     given disableOptimizations; docsCnt is set to the caller's value (merge() leaves it to the application), and the segment is persisted
//     with persist_terms / persist_segment into out_dir (no updated documents).
//   * tref_consider_tracked_sources == MergeCandidatesCollection::consider_tracked_sources over candidates with the given generations.
// Only tests/ and scripts/ load it.
#include "google_codec.h"
#include "indexer.h"
#include "lucene_codec.h"
#include "merge.h"
#include "segment_index_source.h"
#include <chrono>
#include <memory>
#include <string>
#include <vector>

using namespace Trinity;

namespace {
        thread_local std::string g_err;
        thread_local double      g_ms{0};
} // namespace

extern "C" {
const char *tmrg_last_error() {
        return g_err.c_str();
}

// host time of the last tref_merge call's commit() + merge(), one thread
double tmrg_last_ms() {
        return g_ms;
}

// stats[4] = {sumTermHits, totalTerms, sumTermsDocs, docsCnt} as persisted
int tref_merge(int out_codec, const char *out_dir, const char *const *src_dirs, uint32_t n, int disable_optimizations, uint32_t docs_cnt, uint64_t *stats) {
        try {
                std::vector<SegmentIndexSource *>                    srcs;
                std::vector<std::unique_ptr<IndexSourceTermsView>>   views;
                MergeCandidatesCollection                            coll;
                for (uint32_t i = 0; i < n; ++i) {
                        auto s = new SegmentIndexSource(src_dirs[i]);
                        srcs.push_back(s);
                        views.emplace_back(s->segment_terms()->new_terms_view());
                        coll.insert(merge_candidate{s->generation(), views.back().get(), s->access_proxy(), s->masked_documents()});
                }
                std::unique_ptr<Codecs::IndexSession> is;
                if (out_codec == 0)
                        is.reset(new Codecs::Google::IndexSession(out_dir));
                else
                        is.reset(new Codecs::Lucene::IndexSession(out_dir));
                is->begin();
                simple_allocator                               a;
                std::vector<std::pair<str8_t, term_index_ctx>> terms;
                IndexSource::field_statistics                  fs{};
                const auto                                     t0 = std::chrono::steady_clock::now();
                coll.commit();
                coll.merge(is.get(), &a, &terms, &fs, 0, disable_optimizations != 0);
                g_ms       = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
                fs.docsCnt = docs_cnt;
                is->persist_terms(terms);
                std::vector<isrc_docid_t> none;
                persist_segment(fs, is.get(), none);
                if (stats) {
                        stats[0] = fs.sumTermHits;
                        stats[1] = fs.totalTerms;
                        stats[2] = fs.sumTermsDocs;
                        stats[3] = fs.docsCnt;
                }
                for (auto s : srcs)
                        s->Release();
                return 0;
        } catch (const std::exception &e) {
                g_err = e.what();
        } catch (...) {
                g_err = "unknown exception";
        }
        return -1;
}

// out_gens / out_retention[ntracked]: the tracked generations ascending, each with 0 RetainAll, 1 RetainDocumentIDsUpdates, 2 Delete
int tref_consider_tracked_sources(const uint64_t *candidate_gens, uint32_t ncand, const uint64_t *tracked, uint32_t ntracked, uint64_t *out_gens,
                                  uint8_t *out_retention) {
        MergeCandidatesCollection coll;
        for (uint32_t i = 0; i < ncand; ++i)
                coll.insert(merge_candidate{candidate_gens[i], nullptr, nullptr, updated_documents{}});
        const auto r = coll.consider_tracked_sources(std::vector<uint64_t>(tracked, tracked + ntracked));
        for (size_t i = 0; i < r.size(); ++i) {
                out_gens[i]      = r[i].first;
                out_retention[i] = uint8_t(r[i].second);
        }
        return 0;
}
}
