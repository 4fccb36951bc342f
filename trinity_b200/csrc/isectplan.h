// The host step of trn_intersect between its two device passes (engine.cu, intersect.cuh), as a pure function of the distinct masks of
// one request and their first docIDs — so it is pinned on the CPU (trn_debug_intersect_plan, tests/test_intersect_cpu.py).  Host only.
//
// ctx::consider (intersect.cpp:64-91) keeps an array of masks that is the antichain of the maximal masks seen so far: a mask is pushed
// only at its first occurrence, only when no earlier mask is a strict superset of it, and the push swap-removes every strict subset.
// So the array changes only at pushes.  An EPOCH is the stretch of documents from one push to the next; its array, in the order the
// swap-removals leave, follows from the pushes alone, and every considered document of the epoch adds to an entry of that array.
#pragma once
#include <algorithm>
#include <cstdint>
#include <numeric>
#include <string>
#include <unordered_map>
#include <vector>

namespace trn {

static constexpr uint32_t kIsectMaxMasks   = 1u << 16; // distinct masks of one request (TRN_ISECT_MAX_MASKS may lower it)
static constexpr uint64_t kIsectMaxEntries = 1u << 24; // entries of one request's epoch arrays (the sum of the antichain's sizes over its epochs)

struct IsectPlan {
        std::vector<uint32_t> epoch_start; // per epoch: the docID of the push that starts it (ascending)
        std::vector<uint32_t> epoch_off;   // per epoch + 1: its array is entries [epoch_off[e], epoch_off[e + 1])
        std::vector<uint64_t> snap_mask;   // per entry: the mask, in array order
        std::vector<int32_t>  snap_slot;   // per entry: its index in final_mask, -1 when a later push removes it (its count is lost)
        std::vector<uint64_t> final_mask;  // the array after the last document: what the request returns
};

// masks[i] first occurs at docID firsts[i] (distinct masks, any order).  Returns 0, or 1 when there are more than max_masks masks or the
// epoch arrays would hold more than kIsectMaxEntries entries (err says which).
inline int isect_plan(const uint64_t *masks, const uint32_t *firsts, size_t n, uint32_t max_masks, IsectPlan &out, std::string &err) {
        out = IsectPlan{};
        if (n > max_masks) {
                err = std::to_string(n) + " distinct token masks, more than the limit of " + std::to_string(max_masks);
                return 1;
        }
        std::vector<uint32_t> ord(n);
        std::iota(ord.begin(), ord.end(), 0u);
        std::sort(ord.begin(), ord.end(), [&](uint32_t a, uint32_t b) { return firsts[a] < firsts[b]; });
        std::vector<uint64_t> arr;
        out.epoch_off.push_back(0);
        for (const uint32_t k : ord) {
                const uint64_t m = masks[k];
                bool           absorbed{false};
                for (size_t i = 0; i < arr.size();) {
                        const uint64_t v = arr[i];
                        if ((v & m) == m) { // (the array is an antichain: nothing was removed before a superset is met)
                                absorbed = true;
                                break;
                        } else if ((m & v) == v) {
                                arr[i] = arr.back();
                                arr.pop_back();
                        } else
                                ++i;
                }
                if (absorbed)
                        continue;
                arr.push_back(m);
                if (out.snap_mask.size() + arr.size() > kIsectMaxEntries) {
                        err = "the epoch arrays of " + std::to_string(n) + " distinct token masks exceed " + std::to_string(kIsectMaxEntries) + " entries";
                        out = IsectPlan{};
                        return 1;
                }
                out.epoch_start.push_back(firsts[k]);
                out.snap_mask.insert(out.snap_mask.end(), arr.begin(), arr.end());
                out.epoch_off.push_back(uint32_t(out.snap_mask.size()));
        }
        out.final_mask = arr;
        std::unordered_map<uint64_t, int32_t> slot;
        for (size_t i = 0; i < arr.size(); ++i)
                slot.emplace(arr[i], int32_t(i));
        out.snap_slot.resize(out.snap_mask.size());
        for (size_t i = 0; i < out.snap_mask.size(); ++i) {
                const auto it    = slot.find(out.snap_mask[i]);
                out.snap_slot[i] = it == slot.end() ? -1 : it->second;
        }
        return 0;
}

// finalize()'s order made deterministic (intersect.cpp:93-99 sorts by popcount, then count, both descending; ties by mask ascending here)
inline bool isect_result_less(uint64_t ma, uint32_t ca, uint64_t mb, uint32_t cb) {
        const int pa = __builtin_popcountll(ma), pb = __builtin_popcountll(mb);
        if (pa != pb)
                return pa > pb;
        if (ca != cb)
                return ca > cb;
        return ma < mb;
}

} // namespace trn
