// TEST INFRASTRUCTURE — NOT PRODUCT CODE.
//
// C-ABI harness for the reference's indexer (indexer.h, indexer.cpp) with payloads on hits, built by oracle/build_indexer_payloads.sh into
// oracle/_ref/libtrinity_ref_indexer_payloads.so against the reference objects of libtrinity_ref.so (which holds indexer.cpp and both
// codecs).  It drives the reference's own SegmentIndexSession document by document, in the order given, and commit()s the segment into a
// directory:
//   * names[0 .. nterms) are registered with term_id() before the first document, so term t has the transient id t + 1
//   * document d = tokens[doc_offsets[d] .. doc_offsets[d + 1]) at positions[] (null: token i at position i + 1), every token inserted
//     with insert(term, pos, {bytes, len}): the low payload_lens[i] bytes of payloads[i] in memory order
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
const char *tidxp_last_error() {
        return g_err.c_str();
}

// host time of the last tref_index_documents_payloads call: the session's begin / insert / commit, one thread
double tidxp_last_ms() {
        return g_ms;
}

int tref_index_documents_payloads(int codec, const char *dir, const char *const *names, uint32_t nterms, const uint32_t *docids, const uint64_t *doc_offsets,
                                  const uint32_t *tokens, const uint32_t *positions, const uint8_t *payload_lens, const uint64_t *payloads, uint32_t ndocs) {
        try {
                const auto          t0 = std::chrono::steady_clock::now();
                SegmentIndexSession sess;
                for (uint32_t t = 0; t < nterms; ++t)
                        if (sess.term_id(str8_t(names[t], uint8_t(strlen(names[t])))) != t + 1)
                                throw Switch::data_error("names must be distinct");
                for (uint32_t d = 0; d < ndocs; ++d) {
                        auto proxy = sess.begin(docids[d]);
                        for (uint64_t i = doc_offsets[d]; i < doc_offsets[d + 1]; ++i) {
                                uint8_t b[8];
                                std::memcpy(b, &payloads[i], 8);
                                proxy.insert(tokens[i] + 1, tokenpos_t(positions ? positions[i] : i - doc_offsets[d] + 1), {b, payload_lens[i]});
                        }
                        sess.insert(proxy);
                }
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
