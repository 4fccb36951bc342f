// How trn_exec_batch splits a DocumentsOnly / SCORED_ALL batch into pipelined launches (engine.cu), as a pure function of what is known before
// the first launch — so the rule is pinned on the CPU (trn_debug_chunk_plan, tests/test_chunk_plan_cpu.py).  Host only.
#pragma once
#include <algorithm>
#include <cmath>
#include <cstdint>
#include <vector>

namespace trn {

struct ChunkPlanIn {
        uint32_t nq{0};
        bool     topk{false};           // TRN_MODE_SCORED_TOPK: results are nq x k, nothing to pipeline
        uint64_t est_postings{0};       // sum of term.documents over the batch's TERM nodes
        uint64_t leaves{0};             // TERM nodes of the batch
        uint32_t max_chunks{8};         // TRN_PIPELINE_CHUNKS
        uint64_t chunk_postings{1000000000ull}; // first batch of a shape: referenced postings a chunk must carry
        bool     rule_sqrt{true};       // use the result size of the previous batch of this shape when there is one
        bool     taper{true};           // split the last chunk into 1/2, 1/4, 1/4
        double   tail_ms{0.15}, tail_tree_ms{0.9}; // modelled cost of one more launch: conjunction / candidate items, tile items of multi-leaf trees
        uint64_t hint_bytes{0}, hint_postings{0};  // previous host-buffer batch: its result bytes and referenced postings ...
        bool     hint_same_shape{false};           // ... and whether it had this batch's nq and mode
};
struct ChunkPlan {
        bool                  single_call{true}; // one device call + one fetch (no pipelining)
        std::vector<uint32_t> sizes;             // queries per launch, in order (sum == nq)
};

inline ChunkPlan plan_chunks(const ChunkPlanIn &in) {
        ChunkPlan P;
        uint32_t  nchunks  = std::max(1u, in.max_chunks);
        bool      taperOne = false;
        if (nchunks > 1) {
                // a chunk must be worth its launch tails: as many chunks as the referenced postings pay for (a batch of a docID shard holds so
                // little kernel time that eight launches cost more in tails than the overlapped copy saves)
                nchunks = uint32_t(std::min<uint64_t>(nchunks, std::max<uint64_t>(1, in.est_postings / std::max<uint64_t>(1, in.chunk_postings))));
                // With the result size of the previous batch of this shape known, the chunk count balances what chunking buys against what it
                // costs: c chunks (the last one tapered) expose 1/(4c) of the result copy (D ms at ~45 GB/s) and add c + 2 launch tails — minimum
                // at c = sqrt(D / (4 tail)) (engine.cu, trn_exec_batch).
                if (in.rule_sqrt && in.hint_bytes && in.hint_same_shape && in.est_postings >= in.hint_postings - in.hint_postings / 4 &&
                    in.est_postings <= in.hint_postings + in.hint_postings / 4) {
                        const double D    = double(in.hint_bytes) / 45e6; // ms
                        const double tail = in.leaves > 4ull * in.nq ? in.tail_tree_ms : in.tail_ms;
                        nchunks           = uint32_t(std::min<double>(in.max_chunks, std::max(1.0, std::floor(std::sqrt(D / (4.0 * tail)) + 0.5))));
                        // one chunk: still worth its taper (two more launches for 3/4 of the copy off the critical path)?
                        taperOne = in.taper && D > 8.0 / 3.0 * tail;
                }
        }
        if (in.topk || in.nq < 8 * nchunks || (nchunks <= 1 && !(taperOne && in.nq >= 32))) {
                P.sizes.push_back(in.nq);
                return P;
        }
        P.single_call      = false;
        const uint32_t per = (in.nq + nchunks - 1) / nchunks;
        for (uint32_t q0 = 0; q0 < in.nq; q0 += per)
                P.sizes.push_back(std::min(per, in.nq - q0));
        if (in.taper && P.sizes.back() >= 32) {
                // nothing overlaps the LAST chunk's result copy: taper the end of the batch (1/2, 1/4, 1/4 of a chunk) so that what is copied after
                // the last kernel is a quarter of a chunk
                const uint32_t n = P.sizes.back(), a = n / 2, b = n / 4;
                P.sizes.back() = a;
                P.sizes.push_back(b);
                P.sizes.push_back(n - a - b);
        }
        return P;
}

} // namespace trn
