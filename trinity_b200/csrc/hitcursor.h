// Cursors over the positions ("hits") of one document of one term, both codecs — shared by the kernels (phrase.cuh) and the host (the
// CPU tests pin them against the corpus through trn_debug_positions).
//   GOOGLE: Decoder::materialize_hits / skip_block_doc (google_codec.cpp:497-594): hits inline behind a block's freqs
//   LUCENE: refill_hits / materialize_hits (lucene_codec.cpp:401-513, :767-856): hits.data, reached through the load-time hits directory
#pragma once
#include "dirlookup.h"
#include "varbyte.h"
#include <cstdint>

namespace trn {

struct HitTerm { // per term: first entry in hblk_off, sumHits
        uint32_t hb_begin, sum_hits;
};
struct HitsView { // what the cursors read (DevIndex on the device, the host's vectors in the tests)
        const uint8_t * index;
        const uint32_t *blk_last, *blk_off, *tile_first;
        const uint8_t * hits;
        const uint32_t *hit_base, *hblk_off;
        const HitTerm * hit_term;
        int             codec;
};

struct PhraseTerm { // a term of the phrase as the cursor needs it
        uint32_t dir, nb, docs, first, last, tfb, tfbase, tfs;
        uint32_t id;
};

// ---- LUCENE: one int-block (lucene_codec.cpp:69-100 + FastPFor<4> page, fastpfor.h:222-270) read value by value by ONE thread straight
// from global memory (the position check runs a thread per candidate; the warp-cooperative decoders of the scoring kernels do not fit)
TRN_HD uint32_t ldg_u32_unaligned(const uint8_t *p) {
        return uint32_t(TRN_LDG(p)) | (uint32_t(TRN_LDG(p + 1)) << 8) | (uint32_t(TRN_LDG(p + 2)) << 16) | (uint32_t(TRN_LDG(p + 3)) << 24);
}
struct PforRef {
        const uint8_t *pw;    // page word 0 (unaligned); L == 0: the varbyte of the common value
        const uint8_t *pos;   // exception positions (one byte each, ascending)
        const uint8_t *excw;  // packed exception values
        uint32_t       L, b, k, cexcept, same;
        TRN_HD void init(const uint8_t *p) {
                L  = TRN_LDG(p);
                pw = p + 1;
                b = k = cexcept = same = 0;
                pos = excw = nullptr;
                if (L == 0) {
                        const uint8_t *q = pw;
                        same             = varbyte_get(q);
                        return;
                }
                const uint32_t wheremeta = ldg_u32_unaligned(pw + 4);
                b                        = (wheremeta - 1u) >> 2;
                const uint8_t *meta      = pw + (1u + wheremeta) * 4u; // the bytesize word
                const uint32_t bytesize  = ldg_u32_unaligned(meta);
                const uint8_t *bytes     = meta + 4;
                cexcept                  = TRN_LDG(bytes + 1);
                if (cexcept) {
                        k    = uint32_t(TRN_LDG(bytes + 2)) - b;
                        pos  = bytes + 3;
                        excw = meta + 4u + ((bytesize + 3u) & ~3u) + 8u; // past the bitmap word and the count word
                }
        }
        TRN_HD const uint8_t *end() const {
                if (L == 0) {
                        const uint8_t *q = pw;
                        (void)varbyte_get(q);
                        return q;
                }
                return pw + L * 4u;
        }
        // exceptions at positions < i (where a walk that starts at value i finds its first exception)
        TRN_HD uint32_t exceptions_before(uint32_t i) const {
                uint32_t e = 0;
                while (e < cexcept && (uint32_t(TRN_LDG(pos + e)) & 127u) < i)
                        ++e;
                return e;
        }
        // value i of a walk over ascending i; e = the walk's next exception
        TRN_HD uint32_t get(uint32_t i, uint32_t &e) const {
                if (L == 0)
                        return same;
                uint32_t v = 0;
                if (b) {
                        const uint32_t g = i >> 5, j = i & 31u, bp = j * b, wi = 2u + g * b + (bp >> 5), sh = bp & 31u;
                        unsigned long long x = ldg_u32_unaligned(pw + wi * 4u);
                        if (sh + b > 32u)
                                x |= static_cast<unsigned long long>(ldg_u32_unaligned(pw + wi * 4u + 4u)) << 32;
                        v = uint32_t(x >> sh) & (b >= 32u ? 0xffffffffu : ((1u << b) - 1u));
                }
                if (e < cexcept && (uint32_t(TRN_LDG(pos + e)) & 127u) == i) { // out[pos] |= exc << b (fastpfor.h:248-266)
                        uint32_t ev = 1;
                        if (k > 1u) {
                                const uint32_t ebp = e * k, wi = ebp >> 5, esh = ebp & 31u;
                                unsigned long long x = ldg_u32_unaligned(excw + wi * 4u);
                                if (esh + k > 32u)
                                        x |= static_cast<unsigned long long>(ldg_u32_unaligned(excw + wi * 4u + 4u)) << 32;
                                ev = uint32_t(x >> esh) & (k >= 32u ? 0xffffffffu : ((1u << k) - 1u));
                        }
                        v |= b >= 32u ? 0u : (ev << b);
                        ++e;
                }
                return v;
        }
};

// the hits of ONE document of one term: positions are cumulative deltas.
//   GOOGLE (mode 0): inline, a hit = varbyte((delta << 1) | payloadSizeChanged) [u8 size] payload
//   LUCENE (mode 1): inside a 128-hit block of hits.data (int-block of deltas; the payloads sit behind the block, nothing to skip);
//          (mode 2): in the term's varbyte tail, varbyte((delta << 1) | payloadSizeChanged) [u8 size], payloads behind the tail
// A document's run of hits may cross from one block into the next and into the tail.
struct HitCursor {
        const uint8_t *p;
        uint32_t       left; // hits not yet read
        uint32_t       pos;
        uint32_t       psize; // GOOGLE: current payload size (restarts at 0 for every document)
        uint32_t       mode;
        // LUCENE
        const uint8_t * hits;
        const uint32_t *hoff; // the term's hblk_off entries
        uint32_t        hb, nfh, within, e;
        PforRef         blk;
        TRN_HD uint32_t next() {
                --left;
                if (mode == 0u) {
                        const uint32_t step = varbyte_get(p);
                        if (step & 1u)
                                psize = *p++;
                        pos += step >> 1;
                        p += psize;
                        return pos;
                }
                if (mode == 1u) {
                        pos += blk.get(within, e);
                        if (++within == 128u && left) { // on to the next block / the tail
                                ++hb;
                                within = 0;
                                e      = 0;
                                if (hb < nfh)
                                        blk.init(hits + TRN_LDG(hoff + hb));
                                else {
                                        mode = 2u;
                                        p    = hits + TRN_LDG(hoff + nfh);
                                }
                        }
                        return pos;
                }
                const uint32_t step = varbyte_get(p);
                if (step & 1u)
                        ++p; // the new payload size
                pos += step >> 1;
                return pos;
        }
};

// cursor on the hits of document d of the term (left == 0: the term does not hold d)
TRN_HD HitCursor hit_cursor_google(const HitsView &ix, const PhraseTerm &t, uint32_t d) {
        HitCursor c;
        c.p    = nullptr;
        c.left = c.pos = c.psize = c.mode = 0;
        if (!t.nb || d < t.first || d > t.last)
                return c;
        const uint32_t b = dir_first_block_ge(ix.blk_last + t.dir, ix.tile_first + t.tfb, t.nb, t.first, t.last, t.tfbase, t.tfs, d);
        if (b >= t.nb)
                return c;
        const uint32_t last = TRN_LDG(ix.blk_last + t.dir + b), prev = b ? TRN_LDG(ix.blk_last + t.dir + b - 1u) : 0u;
        const uint32_t n    = (b + 1u == t.nb) ? (t.docs - 32u * (t.nb - 1u)) : 32u;
        const uint8_t *p    = ix.index + TRN_LDG(ix.blk_off + t.dir + b); // first doc-delta byte
        // doc deltas: all n-1 of them (the freqs start behind them); the block's last document comes from the directory
        uint32_t idx = 0xffffffffu, doc = prev;
        for (uint32_t i = 0; i + 1u < n; ++i) {
                doc += varbyte_get(p);
                if (doc == d)
                        idx = i;
        }
        if (last == d)
                idx = n - 1u;
        if (idx == 0xffffffffu)
                return c;
        // freqs: the document's own, and (through a second pointer into the same section) those of the documents before it
        const uint8_t *pf   = p;
        uint32_t       mine = 0;
        for (uint32_t i = 0; i < n; ++i) {
                const uint32_t f = varbyte_get(p);
                if (i == idx)
                        mine = f;
        }
        // p is at the block's hits now: skip the hits of the documents before ours
        for (uint32_t i = 0; i < idx; ++i) {
                const uint32_t f = varbyte_get(pf);
                uint32_t       ps = 0;
                for (uint32_t h = 0; h < f; ++h) {
                        const uint32_t step = varbyte_get(p);
                        if (step & 1u)
                                ps = *p++;
                        p += ps;
                }
        }
        c.p    = p;
        c.left = mine & 0xffffu; // freq is uint16_t in the reference (codecs.h:217)
        return c;
}

// LUCENE: cursor on the hits of document d of the term (lucene_codec.cpp:767-856 materialize_hits): the document's index in its
// 128-document block (deltas int-block) and the freqs before it give its first hit's number H = hit_base[block] + sum of those freqs;
// hit H is value H % 128 of the term's (H / 128)-th hit block, or sits in the varbyte tail.
TRN_HD HitCursor hit_cursor_lucene(const HitsView &ix, const PhraseTerm &t, uint32_t d) {
        HitCursor c;
        c.p    = nullptr;
        c.left = c.pos = c.psize = 0;
        c.mode = 1;
        c.hits = ix.hits;
        c.hoff = nullptr;
        c.hb = c.nfh = c.within = c.e = 0;
        if (!t.nb || d < t.first || d > t.last)
                return c;
        const uint32_t b = dir_first_block_ge(ix.blk_last + t.dir, ix.tile_first + t.tfb, t.nb, t.first, t.last, t.tfbase, t.tfs, d);
        if (b >= t.nb)
                return c;
        const uint32_t prev = b ? TRN_LDG(ix.blk_last + t.dir + b - 1u) : 0u;
        const uint8_t *p    = ix.index + TRN_LDG(ix.blk_off + t.dir + b);
        uint32_t       before = 0, mine = 0;
        bool           found = false;
        if (b < (t.docs >> 7)) { // a full block: deltas int-block, freqs int-block
                PforRef D;
                D.init(p);
                uint32_t doc = prev, idx = 0, e = 0;
                for (; idx < 128u; ++idx) {
                        doc += D.get(idx, e);
                        if (doc >= d)
                                break;
                }
                if (idx < 128u && doc == d) {
                        PforRef F;
                        F.init(D.end());
                        e = 0;
                        for (uint32_t i = 0; i < idx; ++i)
                                before += F.get(i, e);
                        mine  = F.get(idx, e);
                        found = true;
                }
        } else { // the tail: (varbyte delta, varbyte freq) pairs (lucene_codec.cpp:527-550)
                const uint32_t n = t.docs & 127u;
                uint32_t       doc = prev;
                for (uint32_t i = 0; i < n && !found; ++i) {
                        doc += varbyte_get(p);
                        const uint32_t f = varbyte_get(p);
                        if (doc == d) {
                                mine  = f;
                                found = true;
                        } else
                                before += f;
                        if (doc > d)
                                break;
                }
        }
        if (!found)
                return c;
        const HitTerm  ht = ix.hit_term[t.id];
        const uint32_t H  = TRN_LDG(ix.hit_base + t.dir + b) + before;
        c.hoff   = ix.hblk_off + ht.hb_begin;
        c.nfh    = ht.sum_hits >> 7;
        c.hb     = H >> 7;
        c.within = H & 127u;
        c.left   = mine & 0xffffu; // freq is uint16_t in the reference (codecs.h:217)
        if (c.hb < c.nfh) {
                c.blk.init(c.hits + TRN_LDG(c.hoff + c.hb));
                c.e = c.blk.exceptions_before(c.within);
        } else { // in the tail: walk to hit `within`
                c.mode = 2;
                c.p    = c.hits + TRN_LDG(c.hoff + c.nfh);
                for (uint32_t i = 0; i < c.within; ++i) {
                        const uint32_t step = varbyte_get(c.p);
                        if (step & 1u)
                                ++c.p;
                }
        }
        return c;
}

TRN_HD HitCursor hit_cursor(const HitsView &ix, const PhraseTerm &t, uint32_t d) {
        return ix.codec == 0 ? hit_cursor_google(ix, t, d) : hit_cursor_lucene(ix, t, d);
}

// ---- hits with their payloads (the default exec mode's term_hit{payload, pos, payloadLen}, runtime.h:8-11; collect.cuh, trn_debug_hits)
// Whether the term holds d at all: a LUCENE document may have freq 0 and so no hits, but the term still holds it.
TRN_HD bool term_holds(const HitsView &ix, const PhraseTerm &t, uint32_t d, uint32_t &freq) {
        freq = 0;
        if (!t.nb || d < t.first || d > t.last)
                return false;
        const uint32_t b = dir_first_block_ge(ix.blk_last + t.dir, ix.tile_first + t.tfb, t.nb, t.first, t.last, t.tfbase, t.tfs, d);
        if (b >= t.nb)
                return false;
        const uint32_t prev = b ? TRN_LDG(ix.blk_last + t.dir + b - 1u) : 0u;
        const uint8_t *p    = ix.index + TRN_LDG(ix.blk_off + t.dir + b);
        if (ix.codec == 0) { // doc deltas, then one freq per document (google_codec.cpp:497-531)
                const uint32_t last = TRN_LDG(ix.blk_last + t.dir + b);
                const uint32_t n    = (b + 1u == t.nb) ? (t.docs - 32u * (t.nb - 1u)) : 32u;
                uint32_t       idx = 0xffffffffu, doc = prev;
                for (uint32_t i = 0; i + 1u < n; ++i) {
                        doc += varbyte_get(p);
                        if (doc == d)
                                idx = i;
                }
                if (last == d)
                        idx = n - 1u;
                if (idx == 0xffffffffu)
                        return false;
                for (uint32_t i = 0; i <= idx; ++i)
                        freq = varbyte_get(p);
                freq &= 0xffffu;
                return true;
        }
        if (b < (t.docs >> 7)) {
                PforRef D;
                D.init(p);
                uint32_t doc = prev, idx = 0, e = 0;
                for (; idx < 128u; ++idx) {
                        doc += D.get(idx, e);
                        if (doc >= d)
                                break;
                }
                if (idx == 128u || doc != d)
                        return false;
                PforRef F;
                F.init(D.end());
                e = F.exceptions_before(idx);
                freq = F.get(idx, e) & 0xffffu;
                return true;
        }
        const uint32_t n   = t.docs & 127u;
        uint32_t       doc = prev;
        for (uint32_t i = 0; i < n; ++i) {
                doc += varbyte_get(p);
                const uint32_t f = varbyte_get(p);
                if (doc == d) {
                        freq = f & 0xffffu;
                        return true;
                }
                if (doc > d)
                        break;
        }
        return false;
}

// low `len` bytes of v replaced by p[0 .. len) (memcpy into the little-endian u64)
TRN_HD uint64_t payload_overwrite(uint64_t v, const uint8_t *p, uint32_t len) {
        uint64_t x = 0;
        for (uint32_t i = 0; i < len; ++i)
                x |= uint64_t(TRN_LDG(p + i)) << (8u * i);
        const uint64_t keep = len >= 8u ? 0ull : (~0ull << (8u * len));
        return (v & keep) | x;
}

// The hits of one document of one term with their payloads, in order:
//   GOOGLE (materialize_hits, google_codec.cpp:533-594): the payload u64 starts at 0 for each document and is zeroed only while the
//          current size is 0; a non-zero size overwrites its low bytes, so a hit keeps the high bytes of an earlier, longer payload.
//   LUCENE (refill_hits / materialize_hits, lucene_codec.cpp:401-462, 767-856): a full 128-hit block is [deltas int-block][payload
//          lengths int-block][varbyte chunk length][payload bytes]; the varbyte tail carries a payload length that persists from hit to
//          hit across documents, starting at 0 at the tail's start, and its payload bytes follow all its varbytes.  Each payload is zeroed
//          before its bytes are copied.
struct HitWalker {
        HitCursor      c;     // positions (its LUCENE block / tail state is followed below)
        uint64_t       payload;
        uint32_t       plen;  // GOOGLE: current size; LUCENE tail: the persisting length
        const uint8_t *pp;    // next payload byte
        PforRef        lens;  // LUCENE full block: payload lengths
        uint32_t       le, tail_n;

        // LUCENE: enter hit block hb at value `within` (lengths of the values before it skipped)
        TRN_HD void lucene_block(uint32_t within) {
                lens.init(c.blk.end());
                const uint8_t *q = lens.end();
                (void)varbyte_get(q); // the chunk length
                pp = q;
                le = 0;
                for (uint32_t i = 0; i < within; ++i)
                        pp += lens.get(i, le);
        }
        // LUCENE: the tail starting at p; position the payload pointer and the persisting length at hit `within`
        TRN_HD void lucene_tail(const uint8_t *p, uint32_t within) {
                uint32_t len = 0, off = 0, at = 0;
                for (uint32_t i = 0; i < tail_n; ++i) {
                        if (i == within)
                                at = len;
                        const uint32_t step = varbyte_get(p);
                        if (step & 1u)
                                len = TRN_LDG(p++);
                        if (i < within)
                                off += len;
                }
                pp   = p + off;
                plen = at;
        }

        TRN_HD void init(const HitsView &ix, const PhraseTerm &t, uint32_t d) {
                c       = hit_cursor(ix, t, d);
                payload = 0;
                plen = le = tail_n = 0;
                pp               = nullptr;
                if (ix.codec == 0 || !c.left)
                        return;
                tail_n = ix.hit_term[t.id].sum_hits & 127u;
                if (c.mode == 1u)
                        lucene_block(c.within);
                else
                        lucene_tail(c.hits + TRN_LDG(c.hoff + c.nfh), c.within);
        }

        // the next hit: returns its position, sets payload / len
        TRN_HD uint32_t next(uint32_t &len) {
                --c.left;
                if (c.mode == 0u) {
                        const uint32_t step = varbyte_get(c.p);
                        if (step & 1u)
                                c.psize = TRN_LDG(c.p++);
                        c.pos += step >> 1;
                        len = c.psize;
                        if (len) {
                                payload = payload_overwrite(payload, c.p, len > 8u ? 8u : len);
                                c.p += len;
                        } else
                                payload = 0;
                        return c.pos;
                }
                if (c.mode == 1u) {
                        c.pos += c.blk.get(c.within, c.e);
                        len     = lens.get(c.within, le);
                        payload = payload_overwrite(0, pp, len > 8u ? 8u : len);
                        pp += len;
                        if (++c.within == 128u && c.left) { // on to the next block / the tail
                                ++c.hb;
                                c.within = 0;
                                c.e      = 0;
                                if (c.hb < c.nfh) {
                                        c.blk.init(c.hits + TRN_LDG(c.hoff + c.hb));
                                        lucene_block(0);
                                } else {
                                        c.mode = 2u;
                                        c.p    = c.hits + TRN_LDG(c.hoff + c.nfh);
                                        lucene_tail(c.p, 0);
                                }
                        }
                        return c.pos;
                }
                const uint32_t step = varbyte_get(c.p);
                if (step & 1u)
                        plen = TRN_LDG(c.p++);
                c.pos += step >> 1;
                len     = plen;
                payload = payload_overwrite(0, pp, len > 8u ? 8u : len);
                pp += len;
                return c.pos;
        }
};


} // namespace trn
