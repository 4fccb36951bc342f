// Segment-directory ingestion (SURVEY.md 8f row 2): reads the files a Trinity SegmentIndexSession::commit() writes
// (indexer.cpp:241-300 persist_segment, terms.cpp:125-170 pack_terms, docidupdates.cpp:8-72 pack_updates) so that the engine runs on
// indexes produced by Trinity's own indexer — the host half of SegmentIndexSource (segment_index_source.cpp:5-186).
//
//   <dir>/index                  raw postings chunks (uploaded to HBM unchanged by trn_upload_index)
//   <dir>/terms.data             { u8 commonPrefixLen, u8 suffixLen, suffix, varuint32 documents, varuint32 chunkLen, u32 chunkOffset }*
//   <dir>/id                     u8 1, u8 len, codec id ("GOOGLE" / "LUCENE"), u64 sumTermHits, u32 totalTerms, u64 sumTermsDocs, u32 docsCnt
//   <dir>/updated_documents.ids  banks of 32K-doc bitmaps [+ 32 KB bloom filter], u8 log2(bank), u8 noBloom, u32 bankBase[], u32 nBanks, u32 lo, u32 hi
// (terms.idx is only a skiplist over terms.data; hits.data holds Lucene positions, which this path never reads.)
#include "../../include/trinity_b200.h"
#include <algorithm>
#include <cerrno>
#include <cstdio>
#include <cstring>
#include <sys/stat.h>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

struct trn_segment {
        int                       codec{0};
        std::vector<uint8_t>      index;
        std::vector<trn_term>     terms;
        std::vector<std::string>  names;
        std::vector<const char *> namePtrs;
        std::vector<uint32_t>     masked;
        uint64_t                  sumTermHits{0}, sumTermsDocs{0};
        uint32_t                  totalTerms{0}, docsCnt{0};
};

namespace {
bool read_file(const std::string &path, std::vector<uint8_t> &out, bool required) {
        std::ifstream f(path, std::ios::binary | std::ios::ate);
        if (!f) {
                if (required)
                        throw std::runtime_error("cannot open " + path);
                return false;
        }
        const std::streamsize n = f.tellg();
        f.seekg(0);
        out.resize(size_t(n));
        if (n && !f.read(reinterpret_cast<char *>(out.data()), n))
                throw std::runtime_error("cannot read " + path);
        return true;
}

// LEB128 as written by Compression::PackUInt32 (Switch/compress.h:65-106)
uint32_t varuint32(const uint8_t *&p, const uint8_t *e) {
        uint32_t v{0};
        for (uint32_t shift = 0; shift < 35; shift += 7) {
                if (p >= e)
                        throw std::runtime_error("terms.data: truncated varuint");
                const uint8_t b = *p++;
                v |= uint32_t(b & 0x7fu) << shift;
                if (b < 128)
                        return v;
        }
        throw std::runtime_error("terms.data: malformed varuint");
}
uint32_t rd32(const uint8_t *p) {
        return p[0] | (uint32_t(p[1]) << 8) | (uint32_t(p[2]) << 16) | (uint32_t(p[3]) << 24);
}
uint64_t rd64(const uint8_t *p) {
        return uint64_t(rd32(p)) | (uint64_t(rd32(p + 4)) << 32);
}
} // namespace

extern "C" int trn_segment_open(const char *dir, trn_segment **out, char *err, size_t errcap) {
        if (!dir || !out)
                return TRN_ERR_ARG;
        auto seg = new trn_segment();
        try {
                const std::string    base(dir);
                std::vector<uint8_t> buf;
                // ---- id: codec + default field statistics
                read_file(base + "/id", buf, true);
                if (buf.size() < 2 || buf[0] != 1 || buf.size() < size_t(2 + buf[1] + 24))
                        throw std::runtime_error("id: unsupported release or truncated");
                const std::string codec(reinterpret_cast<const char *>(buf.data() + 2), buf[1]);
                if (codec == "GOOGLE")
                        seg->codec = TRN_CODEC_GOOGLE;
                else if (codec == "LUCENE")
                        seg->codec = TRN_CODEC_LUCENE;
                else
                        throw std::runtime_error("id: unknown codec '" + codec + "'");
                const uint8_t *p  = buf.data() + 2 + buf[1];
                seg->sumTermHits  = rd64(p);
                seg->totalTerms   = rd32(p + 8);
                seg->sumTermsDocs = rd64(p + 12);
                seg->docsCnt      = rd32(p + 20);
                // ---- index
                read_file(base + "/index", seg->index, true);
                // ---- terms.data: front-coded dictionary, every term carries its term_index_ctx
                if (read_file(base + "/terms.data", buf, false)) {
                        const uint8_t *q = buf.data(), *const e = q + buf.size();
                        std::string    prev;
                        while (q < e) {
                                if (q + 2 > e)
                                        throw std::runtime_error("terms.data: truncated entry");
                                const uint32_t common = q[0], suffix = q[1];
                                q += 2;
                                if (common > prev.size() || q + suffix > e)
                                        throw std::runtime_error("terms.data: bad prefix/suffix lengths");
                                std::string term = prev.substr(0, common) + std::string(reinterpret_cast<const char *>(q), suffix);
                                q += suffix;
                                trn_term t;
                                t.documents = varuint32(q, e);
                                t.chunk_len = varuint32(q, e);
                                if (q + 4 > e)
                                        throw std::runtime_error("terms.data: truncated chunk offset");
                                t.chunk_off = rd32(q);
                                q += 4;
                                if (uint64_t(t.chunk_off) + t.chunk_len > seg->index.size())
                                        throw std::runtime_error("terms.data: chunk of '" + term + "' exceeds the index file");
                                seg->terms.push_back(t);
                                seg->names.push_back(term);
                                prev.swap(term);
                        }
                }
                seg->namePtrs.reserve(seg->names.size());
                for (auto &n : seg->names)
                        seg->namePtrs.push_back(n.c_str());
                // ---- updated_documents.ids: the docIDs this (newer) segment masks in OLDER segments
                if (read_file(base + "/updated_documents.ids", buf, false) && !buf.empty()) {
                        if (buf.size() < 14)
                                throw std::runtime_error("updated_documents.ids: truncated trailer");
                        const uint8_t *e      = buf.data() + buf.size();
                        const uint32_t nbanks = rd32(e - 12);
                        const uint8_t *skip   = e - 12 - size_t(nbanks) * 4;
                        if (skip - 2 < buf.data())
                                throw std::runtime_error("updated_documents.ids: bad skiplist size");
                        const uint32_t bankBits = 1u << skip[-2];
                        const bool     noBloom  = skip[-1] != 0;
                        const size_t   bankBytes = bankBits / 8;
                        const size_t   need      = size_t(nbanks) * bankBytes + (noBloom ? 0 : 256 * 1024 / 8);
                        if (size_t(skip - 2 - buf.data()) != need)
                                throw std::runtime_error("updated_documents.ids: size does not match its trailer");
                        for (uint32_t b = 0; b < nbanks; ++b) {
                                const uint32_t bankBase = rd32(skip + size_t(b) * 4);
                                const uint8_t *bm       = buf.data() + size_t(b) * bankBytes;
                                for (uint32_t i = 0; i < bankBits; ++i)
                                        if (bm[i >> 3] & (1u << (i & 7)))
                                                seg->masked.push_back(bankBase + i);
                        }
                }
                *out = seg;
                return TRN_OK;
        } catch (const std::exception &ex) {
                if (err && errcap) {
                        std::strncpy(err, ex.what(), errcap - 1);
                        err[errcap - 1] = 0;
                }
                delete seg;
                return TRN_ERR_FORMAT;
        }
}

// ---- segment writer: the files of persist_segment (indexer.cpp:241-300) + IndexSession::persist_terms (codecs.cpp:17-27)
namespace {
void put_varuint32(std::vector<uint8_t> &b, uint32_t v) { // == Compression::PackUInt32 (LEB128)
        while (v >= 128) {
                b.push_back(uint8_t(v | 0x80u));
                v >>= 7;
        }
        b.push_back(uint8_t(v));
}
void put32(std::vector<uint8_t> &b, uint32_t v) {
        for (int i = 0; i < 4; ++i)
                b.push_back(uint8_t(v >> (8 * i)));
}
void put64(std::vector<uint8_t> &b, uint64_t v) {
        put32(b, uint32_t(v));
        put32(b, uint32_t(v >> 32));
}
// through <name>.t + rename, as the reference persists `index` and `hits.data`
void write_file(const std::string &path, const uint8_t *p, size_t n) {
        const std::string tmp = path + ".t";
        FILE *            f   = std::fopen(tmp.c_str(), "wb");
        if (!f)
                throw std::runtime_error("cannot create " + tmp);
        const bool ok = (!n || std::fwrite(p, 1, n, f) == n);
        if (std::fclose(f) != 0 || !ok) {
                std::remove(tmp.c_str());
                throw std::runtime_error("cannot write " + tmp);
        }
        if (std::rename(tmp.c_str(), path.c_str()) != 0) {
                std::remove(tmp.c_str());
                throw std::runtime_error("cannot rename " + tmp);
        }
}
struct arg_error : std::runtime_error {
        using std::runtime_error::runtime_error;
};
} // namespace

extern "C" int trn_segment_write(const char *dir, int codec, const uint8_t *index, uint64_t index_bytes, const uint8_t *hits, uint64_t hits_bytes,
                                 const trn_term *terms, const char *const *names, uint32_t nterms, uint64_t sum_term_hits, uint32_t total_terms,
                                 uint64_t sum_terms_docs, uint32_t docs_cnt, const uint32_t *updated_docids, uint64_t nupdated, char *err, size_t errcap) {
        const auto say = [&](const char *m) {
                if (err && errcap) {
                        std::strncpy(err, m, errcap - 1);
                        err[errcap - 1] = 0;
                }
        };
        try {
                if (!dir || (codec != TRN_CODEC_GOOGLE && codec != TRN_CODEC_LUCENE) || (index_bytes && !index) || (hits_bytes && !hits) || (nterms && (!terms || !names)) ||
                    (nupdated && !updated_docids))
                        throw arg_error("trn_segment_write: bad arguments");
                std::string base(dir);
                while (base.size() > 1 && base.back() == '/')
                        base.pop_back();
                const std::string last = base.substr(base.find_last_of('/') == std::string::npos ? 0 : base.find_last_of('/') + 1);
                if (last.empty() || last.find_first_not_of("0123456789") != std::string::npos)
                        throw arg_error("trn_segment_write: the last component of '" + base + "' must be a number, the segment's generation");
                // ---- the dictionary: terms that have documents, in terms_cmp order (bytewise, the shorter first: common.h:48-57)
                std::vector<uint32_t> order;
                for (uint32_t i = 0; i < nterms; ++i) {
                        const size_t len = names[i] ? std::strlen(names[i]) : 0;
                        if (len == 0 || len > 64)
                                throw arg_error("trn_segment_write: term " + std::to_string(i) + ": a name has 1 .. 64 bytes (Limits::MaxTermLength), this one " +
                                                std::to_string(len));
                        if (terms[i].documents)
                                order.push_back(i);
                }
                std::vector<uint32_t> all(nterms);
                for (uint32_t i = 0; i < nterms; ++i)
                        all[i] = i;
                const auto by_name = [&](uint32_t a, uint32_t b) { return std::strcmp(names[a], names[b]) < 0; };
                std::sort(all.begin(), all.end(), by_name);
                for (uint32_t i = 1; i < nterms; ++i)
                        if (!std::strcmp(names[all[i - 1]], names[all[i]]))
                                throw arg_error("trn_segment_write: terms " + std::to_string(std::min(all[i - 1], all[i])) + " and " +
                                                std::to_string(std::max(all[i - 1], all[i])) + " have the same name '" + names[all[i]] + "'");
                std::sort(order.begin(), order.end(), by_name);
                // ---- updated_documents.ids (pack_updates, docidupdates.cpp:8-73)
                std::vector<uint8_t> upd;
                if (nupdated) {
                        std::vector<uint32_t> ids(updated_docids, updated_docids + nupdated);
                        std::sort(ids.begin(), ids.end());
                        for (size_t i = 1; i < ids.size(); ++i)
                                if (ids[i] == ids[i - 1])
                                        throw arg_error("trn_segment_write: docID " + std::to_string(ids[i]) + " is updated twice (Already committed document, indexer.cpp:219-222)");
                        constexpr size_t   BANK = 32 * 1024, BLOOM = 256 * 1024;
                        const bool         bloom = ids.size() > BANK * 8;
                        std::vector<uint8_t> bf(bloom ? BLOOM / 8 : 0, 0), skip;
                        for (size_t i = 0; i < ids.size();) {
                                const uint32_t bank = ids[i];
                                const uint64_t upto = uint64_t(bank) + BANK;
                                const size_t   at   = upd.size();
                                upd.resize(at + BANK / 8, 0);
                                put32(skip, bank);
                                for (; i < ids.size() && ids[i] < upto; ++i) {
                                        const uint32_t rel = ids[i] - bank, h = ids[i] & uint32_t(BLOOM - 1);
                                        if (bloom)
                                                bf[h >> 3] |= uint8_t(1u << (h & 7));
                                        upd[at + (rel >> 3)] |= uint8_t(1u << (rel & 7));
                                }
                        }
                        upd.insert(upd.end(), bf.begin(), bf.end());
                        upd.push_back(15); // log2(BANK)
                        upd.push_back(bloom ? 0 : 1);
                        const uint32_t nbanks = uint32_t(skip.size() / 4);
                        upd.insert(upd.end(), skip.begin(), skip.end());
                        put32(upd, nbanks);
                        put32(upd, ids.front());
                        put32(upd, ids.back());
                }
                // ---- terms.data / terms.idx (pack_terms, terms.cpp:126-172): one skiplist entry per 64 terms, the first term always
                std::vector<uint8_t> data, idx;
                uint32_t             next{1};
                std::string          prev;
                for (const uint32_t i : order) {
                        const std::string cur(names[i]);
                        if (--next == 0) {
                                next = 64;
                                idx.push_back(uint8_t(cur.size()));
                                idx.insert(idx.end(), cur.begin(), cur.end());
                                put_varuint32(idx, uint32_t(data.size()));
                        }
                        size_t common{0};
                        while (common < cur.size() && common < prev.size() && cur[common] == prev[common])
                                ++common;
                        data.push_back(uint8_t(common));
                        data.push_back(uint8_t(cur.size() - common));
                        data.insert(data.end(), cur.begin() + common, cur.end());
                        put_varuint32(data, terms[i].documents);
                        put_varuint32(data, terms[i].chunk_len);
                        put32(data, terms[i].chunk_off);
                        prev = cur;
                }
                // ---- id: release 1, the codec's name, the default field's statistics
                std::vector<uint8_t> id{1, 6};
                for (const char ch : std::string(codec == TRN_CODEC_GOOGLE ? "GOOGLE" : "LUCENE"))
                        id.push_back(uint8_t(ch));
                put64(id, sum_term_hits);
                put32(id, total_terms);
                put64(id, sum_terms_docs);
                put32(id, docs_cnt);
                try {
                        if (::mkdir(base.c_str(), 0775) != 0 && errno != EEXIST)
                                throw std::runtime_error("cannot create " + base);
                        write_file(base + "/terms.data", data.data(), data.size());
                        write_file(base + "/terms.idx", idx.data(), idx.size());
                        if (!upd.empty())
                                write_file(base + "/updated_documents.ids", upd.data(), upd.size());
                        write_file(base + "/id", id.data(), id.size());
                        if (codec == TRN_CODEC_LUCENE && hits_bytes)
                                write_file(base + "/hits.data", hits, hits_bytes);
                        write_file(base + "/index", index, index_bytes);
                } catch (const std::exception &ex) {
                        say(ex.what());
                        return TRN_ERR_STATE;
                }
                return TRN_OK;
        } catch (const arg_error &ex) {
                say(ex.what());
                return TRN_ERR_ARG;
        } catch (const std::exception &ex) {
                say(ex.what());
                return TRN_ERR_STATE;
        }
}

extern "C" void trn_segment_close(trn_segment *s) {
        delete s;
}

extern "C" int trn_segment_info(trn_segment *s, int *codec, uint32_t *nterms, uint64_t *index_bytes, uint64_t *sum_term_hits, uint32_t *total_terms,
                                uint64_t *sum_terms_docs, uint32_t *docs_cnt, uint64_t *nmasked) {
        if (!s)
                return TRN_ERR_ARG;
        if (codec) *codec = s->codec;
        if (nterms) *nterms = uint32_t(s->terms.size());
        if (index_bytes) *index_bytes = s->index.size();
        if (sum_term_hits) *sum_term_hits = s->sumTermHits;
        if (total_terms) *total_terms = s->totalTerms;
        if (sum_terms_docs) *sum_terms_docs = s->sumTermsDocs;
        if (docs_cnt) *docs_cnt = s->docsCnt;
        if (nmasked) *nmasked = s->masked.size();
        return TRN_OK;
}

extern "C" int trn_segment_index(trn_segment *s, const uint8_t **index, uint64_t *nbytes) {
        if (!s || !index || !nbytes)
                return TRN_ERR_ARG;
        *index  = s->index.data();
        *nbytes = s->index.size();
        return TRN_OK;
}

extern "C" int trn_segment_terms(trn_segment *s, const trn_term **terms, const char *const **names, uint32_t *nterms) {
        if (!s || !terms || !names || !nterms)
                return TRN_ERR_ARG;
        *terms  = s->terms.data();
        *names  = s->namePtrs.data();
        *nterms = uint32_t(s->terms.size());
        return TRN_OK;
}

extern "C" int trn_segment_masked(trn_segment *s, const uint32_t **docids, uint64_t *n) {
        if (!s || !docids || !n)
                return TRN_ERR_ARG;
        *docids = s->masked.data();
        *n      = s->masked.size();
        return TRN_OK;
}
