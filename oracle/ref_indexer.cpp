// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's indexer (indexer.h, indexer.cpp), built by oracle/build_indexer.sh into
// oracle/_ref/libtrinity_ref_indexer.so against the reference objects of libtrinity_ref.so (which holds indexer.cpp and both codecs).
// It drives the reference's own SegmentIndexSession document by document, in the order given, with explicit positions, and commit()s the
// segment into a directory:
//   * names[0 .. nterms) are registered with term_id() before the first document, so term t has the transient id t + 1
//   * document d = tokens[doc_offsets[d] .. doc_offsets[d + 1]) at positions[] (null: token i at position i + 1), inserted in the order
//     given; replace_flags[d] != 0 (may be null): committed with replace() instead of insert()
//   * erased[0 .. nerased): erase()d after the documents
// Only tests/ and scripts/ load it.
#include "google_codec.h"
#include "indexer.h"
#include "lucene_codec.h"
#include <chrono>
#include <cstring>
#include <string>

using namespace Trinity;

namespace {
        thread_local std::string g_err;
        thread_local double      g_ms{0};
} // namespace

extern "C" {
const char *tidx_last_error() {
        return g_err.c_str();
}

// host time of the last tref_index_documents call: the session's begin / insert / commit, one thread
double tidx_last_ms() {
        return g_ms;
}

int tref_index_documents(int codec, const char *dir, const char *const *names, uint32_t nterms, const uint32_t *docids, const uint64_t *doc_offsets,
                         const uint32_t *tokens, const uint32_t *positions, uint32_t ndocs, const uint8_t *replace_flags, const uint32_t *erased, uint32_t nerased) {
        try {
                const auto          t0 = std::chrono::steady_clock::now();
                SegmentIndexSession sess;
                for (uint32_t t = 0; t < nterms; ++t)
                        if (sess.term_id(str8_t(names[t], uint8_t(strlen(names[t])))) != t + 1)
                                throw Switch::data_error("names must be distinct");
                for (uint32_t d = 0; d < ndocs; ++d) {
                        auto proxy = sess.begin(docids[d]);
                        for (uint64_t i = doc_offsets[d]; i < doc_offsets[d + 1]; ++i)
                                proxy.insert(tokens[i] + 1, tokenpos_t(positions ? positions[i] : i - doc_offsets[d] + 1));
                        if (replace_flags && replace_flags[d])
                                sess.replace(proxy);
                        else
                                sess.insert(proxy);
                }
                for (uint32_t i = 0; i < nerased; ++i)
                        sess.erase(erased[i]);
                if (codec == 0) {
                        Codecs::Google::IndexSession cs(dir);
                        sess.commit(&cs);
                } else {
                        Codecs::Lucene::IndexSession cs(dir);
                        sess.commit(&cs);
                }
                g_ms = std::chrono::duration<double, std::milli>(std::chrono::steady_clock::now() - t0).count();
                return 0;
        } catch (const std::exception &e) {
                g_err = e.what();
        } catch (...) {
                g_err = "unknown exception";
        }
        return -1;
}
}
