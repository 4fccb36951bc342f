// Host-side write path for the two on-disk postings layouts the GPU engine reads.
// The interface mirrors the reference plugin API (codecs.h:57-200: IndexSession / Encoder,
// begin_term / begin_document / new_hit / end_document / end_term) so that callers and tests
// read like the reference's; the bytes produced are identical to the reference encoders'
// (google_codec.cpp:9-176, lucene_codec.cpp:163-388 + FastPFor<4> fastpfor.h:167-220) — pinned
// byte-for-byte by tests/test_codecs_cpu.py against oracle/_ref.
#pragma once
#include <cstddef>
#include <cstdint>
#include <vector>

namespace trn {

// == Trinity::term_index_ctx (codecs.h:17-55): {documents, indexChunk{offset,len}}
struct term_index_ctx {
        uint32_t documents{0};
        uint32_t offset{0};
        uint32_t size{0};
};

enum class Codec : int { Google = 0, Lucene = 1 };

namespace Codecs {

        // == Trinity::Codecs::IndexSession (codecs.h:66-173): owns indexOut (+ positionsOut for Lucene == hits.data)
        struct IndexSession {
                const Codec          codec;
                std::vector<uint8_t> indexOut;
                std::vector<uint8_t> positionsOut; // Lucene only (hits.data)

                explicit IndexSession(Codec c)
                    : codec{c} {
                }
                const char *codec_identifier() const {
                        return codec == Codec::Google ? "GOOGLE" : "LUCENE";
                }
        };

        // == Trinity::Codecs::Encoder (codecs.h:176-200)
        struct Encoder {
                IndexSession *const sess;
                explicit Encoder(IndexSession *s)
                    : sess{s} {
                }
                virtual ~Encoder() = default;
                virtual void begin_term()                                                                      = 0;
                virtual void begin_document(uint32_t documentID)                                               = 0;
                virtual void new_hit(uint32_t position, const uint8_t *payload = nullptr, uint8_t payloadSize = 0) = 0;
                virtual void end_document()                                                                    = 0;
                virtual void end_term(term_index_ctx *out)                                                     = 0;
        };

        namespace Google {
                static constexpr uint32_t N{32};                  // docs per block (google_codec.h:18)
                static constexpr uint32_t MAX_N{128};             // largest block size the decode sweep (BASELINE configs[4]) builds
                static constexpr uint32_t SKIPLIST_STEP{256 / N}; // one skiplist entry every 8 blocks (google_codec.h:19)

                class Encoder final : public Codecs::Encoder {
                        std::vector<uint8_t> skipListData, block, hitsData;
                        uint32_t             prevBlockLastDocumentID{0}, curDocID{0}, lastCommitedDocID{0};
                        uint32_t             curBlockSize{0};
                        uint8_t              curPayloadSize{0};
                        uint32_t             lastPos{0};
                        uint32_t             docDeltas[MAX_N];
                        uint32_t             blockFreqs[MAX_N];
                        uint32_t             curTermOffset{0};
                        uint32_t             termDocuments{0};
                        void                 commit_block();

                      public:
                        // NOT reset per term in the reference (google_codec.h:57, google_codec.cpp:9-23): the phase of the
                        // first skiplist entry of a term depends on how many blocks earlier terms committed.
                        uint32_t skiplistEntryCountdown{SKIPLIST_STEP};
                        // the two compile-time constants of google_codec.h:17-20 as run-time values — ONLY for the decode sweep
                        // (BASELINE.json configs[4]: block size / skiplist step vs HBM GB/s); the reference format is {32, 8}
                        uint32_t blockDocs{N}, skiplistStep{SKIPLIST_STEP};

                        explicit Encoder(IndexSession *s)
                            : Codecs::Encoder{s} {
                        }
                        void begin_term() override;
                        void begin_document(uint32_t documentID) override;
                        void new_hit(uint32_t position, const uint8_t *payload = nullptr, uint8_t payloadSize = 0) override;
                        void end_document() override;
                        void end_term(term_index_ctx *out) override;
                };
        } // namespace Google

        namespace Lucene {
                static constexpr uint32_t BLOCK_SIZE{128};  // lucene_codec.h:54
                static constexpr uint32_t SKIPLIST_STEP{1}; // lucene_codec.h:57

                // one int-block (lucene_codec.cpp:26-66): u8 0 + varbyte(v) if all equal, else u8 L + L x u32 FastPFor<4> page
                void ints_encode(const uint32_t *values, std::vector<uint8_t> &out);

                class Encoder final : public Codecs::Encoder {
                        struct skiplist_entry {
                                uint32_t indexOffset, lastDocID, lastHitsBlockOffset, totalDocumentsSoFar, lastHitsBlockTotalHits;
                                uint16_t curHitsBlockHits;
                        };
                        std::vector<skiplist_entry> skiplist;
                        skiplist_entry              cur_block{};
                        uint32_t                    docDeltas[BLOCK_SIZE], docFreqs[BLOCK_SIZE], hitPosDeltas[BLOCK_SIZE], hitPayloadSizes[BLOCK_SIZE];
                        std::vector<uint8_t>        payloadsBuf;
                        uint32_t                    lastDocID{0}, lastPosition{0}, totalHits{0}, sumHits{0}, buffered{0}, termDocuments{0};
                        uint32_t                    termIndexOffset{0}, termPositionsOffset{0}, lastHitsBlockOffset{0}, lastHitsBlockTotalHits{0};
                        uint32_t                    skiplistCountdown{SKIPLIST_STEP};
                        void                        output_block();

                      public:
                        explicit Encoder(IndexSession *s)
                            : Codecs::Encoder{s} {
                        }
                        void begin_term() override;
                        void begin_document(uint32_t documentID) override;
                        void new_hit(uint32_t position, const uint8_t *payload = nullptr, uint8_t payloadSize = 0) override;
                        void end_document() override;
                        void end_term(term_index_ctx *out) override;
                };
        } // namespace Lucene

        Encoder *new_encoder(IndexSession *s);

} // namespace Codecs

// ---------------------------------------------------------------------------------------------------------
// Load-time block directory (replaces the per-query skiplist parse of Decoder::init, google_codec.cpp:936-983 /
// lucene_codec.cpp:877-932, and the header hops of seek_block google_codec.cpp:641-697).  One entry per block:
//   blk_last[i] = last docID of block i;  blk_off[i] = byte offset (from index base) of the block's first payload
//   byte (Google: first doc-delta varbyte, after the n byte; Lucene: the u8 L of the deltas int-block / the first
//   varbyte of the tail).  Each term owns nblocks+1 consecutive entries; the sentinel entry holds
//   {last = UINT32_MAX, off = end of the term's block area}.
//
// Sparse docID -> block index on top of it (the O(1) part of skiplist_search, google_codec.cpp:464-495 / lucene_codec.cpp:596-656):
// a term with more than kDirNoTableBlocks blocks owns tf_n + 1 entries of `tile_first`, entry j = first block whose last docID is
// >= (tf_base + j) << tf_shift.  The entries cover only [first_doc, last_doc] of the term (inside THIS index source: a docID-range
// shard indexes its own range), and tf_shift is the smallest granularity >= kDirMinShift that keeps the table at or below one entry
// per kDirBlocksPerEntry blocks — so the whole directory is O(blocks + terms), never terms x tiles.  A lookup reads two neighbouring
// entries and finishes with a binary search over the blk_last entries between them (dependent loads: they were the
// top stall of the candidate probes when a frequent term had 128 blocks per 8192-document entry, hence the finer granularity: a term
// with 64 docIDs per block gets 512-docID entries = 8 blocks = 3 steps); smaller terms (tf_shift == kDirNoTable) search all of blk_last.
static constexpr uint32_t kDirMinShift       = 9;
static constexpr uint32_t kDirBlocksPerEntry = 2;
static constexpr uint32_t kDirNoTable       = 32; // tf_shift value of a term without table
static constexpr uint32_t kDirNoTableBlocks = 8;

struct TermDir {
        uint32_t documents;
        uint32_t dir_begin; // index of the term's first entry in blk_last/blk_off
        uint32_t nblocks;   // excluding sentinel
        uint32_t first_doc, last_doc;
        uint32_t tf_begin{0}, tf_base{0}, tf_shift{kDirNoTable}, tf_n{0};
};

struct BlockDirectory {
        std::vector<uint32_t> blk_last, blk_off, tile_first;
        std::vector<TermDir>  terms;
        uint32_t              block_docs{0}; // documents per full block: GOOGLE 32 (what the terms' blocks say; other values come from the decode sweep), LUCENE 128
        uint64_t              bytes() const { // what the device copy occupies (DevTerm = 36 B per term)
                return (blk_last.size() + blk_off.size() + tile_first.size()) * 4ull + terms.size() * 36ull;
        }
};

// LUCENE positions (lucene_codec.cpp:401-513 refill_hits / :767-856 materialize_hits): a term's hits live in hits.data, 128 per PFor
// block (position deltas int-block, payload sizes int-block, varbyte payload length, payloads) + a varbyte tail, documents owning
// consecutive runs of freq(doc) hits.  The reference reaches a document's hits through the skiplist entry of its block
// ({hits block offset, hits already consumed}, one entry per block for <= 65535 blocks) and by decoding forward; here, like the block
// directory, every block gets its entry at load time:
//   hit_base[dir_begin + b] = hits owned by the term's documents before block b (sentinel entry: the term's sumHits), and
//   hblk_off[hb_begin + h]  = byte offset in hits.data of the term's h-th 128-hit block; entry nfull = the varbyte tail, entry nfull + 1 = its end.
struct HitsDirectory {
        std::vector<uint32_t> hit_base, hblk_off;
        std::vector<uint32_t> hb_begin, sum_hits; // per term
        uint64_t              bytes() const {
                return (hit_base.size() + hblk_off.size() + hb_begin.size() + sum_hits.size()) * 4ull;
        }
};
// throws std::runtime_error on malformed chunks / hit streams
void build_hits_directory(const uint8_t *index, uint64_t nbytes, const uint8_t *hits, uint64_t hbytes, const term_index_ctx *terms, uint32_t nterms,
                          const BlockDirectory &dir, int threads, HitsDirectory &out);

// throws std::runtime_error on malformed chunks
void build_block_directory(Codec codec, const uint8_t *index, uint64_t nbytes, const term_index_ctx *terms, uint32_t nterms, int threads, BlockDirectory &out);

} // namespace trn
