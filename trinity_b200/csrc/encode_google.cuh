// GPU-side Encoder for the GOOGLE postings layout (SURVEY.md 8(f) row 4: "index build on device").  (Included by kernels.cu.)
//
// Replaces (reference): Codecs::Google::Encoder begin_term / begin_document / new_hit / end_document / commit_block / end_term
// (google_codec.cpp:9-176) — the byte stream is the one that encoder writes, pinned bit for bit by tests/test_gpu_encoder.py (no payloads)
// and tests/test_gpu_payloads.py (payloads) against this repo's host encoder (itself pinned against the reference's, tests/test_codecs_cpu.py,
// tests/test_payloads_cpu.py) and against reference-authored indexes.
//
// The reference's encoder is a serial state machine; what makes the layout parallel is that a block's bytes depend on nothing but its own
// documents and the docID right before it:
//   block   = varbyte(last docID - previous block's last docID) varbyte(blockLength) u8 n | n-1 varbyte docID deltas | n varbyte freqs | hits
//   hits    = for every hit of every document, in order: varbyte((pos - previous pos of the document) << 1)          (no payload)
//             with payloads (the PAYLOADS instantiation): varbyte(delta << 1 | changed) [u8 size when changed] payload bytes, `changed` =
//             the size differs from the previous hit's of the same document (0 before its first hit, google_codec.cpp:34, 59-68)
//   chunk   = u16 skiplist entries | blocks | entries x {u32 previous block's last docID, u32 block offset from the chunk start}
//   an entry is written for the block whose commit makes the session-wide countdown hit 0 (every SKIPLIST_STEP-th committed block,
//   counted ACROSS terms, google_codec.h:57), at most 65535 per term.
// so: (1) one warp per block computes the block's size, (2) an exclusive scan of the sizes places every block, (3) one warp per block
// writes it.  Input arrays are read coalesced (lane = document); output bytes of neighbouring lanes are neighbouring bytes.
#pragma once

static constexpr uint32_t kEncScanSpan = 4096; // entries per CTA of the scan kernels (256 threads x 16)

__device__ __forceinline__ uint32_t vb_len_of(uint32_t x) {
        return x < (1u << 7) ? 1u : x < (1u << 14) ? 2u : x < (1u << 21) ? 3u : x < (1u << 28) ? 4u : 5u;
}
__device__ __forceinline__ uint8_t *vb_store(uint8_t *p, uint32_t x) { // == varbyte_put (varbyte.h; Switch/switch_compiler_aux.h:23-81)
        if (x < (1u << 7)) {
                p[0] = uint8_t(x);
                return p + 1;
        }
        if (x < (1u << 14)) {
                p[0] = uint8_t(0x80u | (x >> 8));
                p[1] = uint8_t(x);
                return p + 2;
        }
        if (x < (1u << 21)) {
                p[0] = uint8_t(0xc0u | (x >> 16));
                p[1] = uint8_t(x);
                p[2] = uint8_t(x >> 8);
                return p + 3;
        }
        if (x < (1u << 28)) {
                p[0] = uint8_t(0xe0u | (x >> 24));
                p[1] = uint8_t(x >> 16);
                p[2] = uint8_t(x >> 8);
                p[3] = uint8_t(x);
                return p + 4;
        }
        p[0] = 0xf0u;
        p[1] = uint8_t(x);
        p[2] = uint8_t(x >> 8);
        p[3] = uint8_t(x >> 16);
        p[4] = uint8_t(x >> 24);
        return p + 5;
}

// ---- exclusive scan u32 -> u64 over up to 2^40 entries: partial sums per 4096-entry span, one CTA scans the partials, spans rescanned
__global__ void __launch_bounds__(256) k_enc_scan_partials(const uint32_t *in, uint64_t n, unsigned long long *partials) {
        __shared__ unsigned long long s_w[8];
        const uint64_t base = uint64_t(blockIdx.x) * kEncScanSpan;
        unsigned long long s = 0;
#pragma unroll
        for (uint32_t k = 0; k < 16; ++k) {
                const uint64_t i = base + k * 256u + threadIdx.x;
                s += i < n ? in[i] : 0u;
        }
        for (int o = 16; o; o >>= 1)
                s += __shfl_xor_sync(0xffffffffu, s, o);
        if ((threadIdx.x & 31) == 0)
                s_w[threadIdx.x >> 5] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
                unsigned long long t = 0;
                for (int w = 0; w < 8; ++w)
                        t += s_w[w];
                partials[blockIdx.x] = t;
        }
}

__global__ void __launch_bounds__(1024) k_enc_scan_top(unsigned long long *partials, uint32_t nparts) { // in place -> exclusive; partials[nparts] = total
        __shared__ unsigned long long s_t[1024];
        const uint32_t per = (nparts + 1023u) / 1024u, b = threadIdx.x * per, e = min(nparts, b + per);
        unsigned long long s = 0;
        for (uint32_t i = b; i < e; ++i)
                s += partials[i];
        s_t[threadIdx.x] = s;
        __syncthreads();
        if (threadIdx.x == 0) {
                unsigned long long run = 0;
                for (int i = 0; i < 1024; ++i) {
                        const unsigned long long v = s_t[i];
                        s_t[i]                     = run;
                        run += v;
                }
                partials[nparts] = run;
        }
        __syncthreads();
        unsigned long long run = s_t[threadIdx.x];
        for (uint32_t i = b; i < e; ++i) {
                const unsigned long long v = partials[i];
                partials[i]                = run;
                run += v;
        }
}

__global__ void __launch_bounds__(256) k_enc_scan_final(const uint32_t *in, uint64_t n, const unsigned long long *partials, uint32_t nparts, unsigned long long *out) {
        __shared__ unsigned long long s_w[8];
        __shared__ unsigned long long s_run;
        const uint64_t base = uint64_t(blockIdx.x) * kEncScanSpan;
        const int      lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
        if (threadIdx.x == 0)
                s_run = partials[blockIdx.x];
        if (blockIdx.x == 0 && threadIdx.x == 0)
                out[n] = partials[nparts];
        __syncthreads();
        for (uint32_t k = 0; k < 16; ++k) {
                const uint64_t     i = base + k * 256u + threadIdx.x;
                const uint32_t     v = i < n ? in[i] : 0u;
                unsigned long long x = v;
                for (int o = 1; o < 32; o <<= 1) {
                        const unsigned long long y = __shfl_up_sync(0xffffffffu, x, o);
                        if (lane >= o)
                                x += y;
                }
                if (lane == 31)
                        s_w[warp] = x;
                __syncthreads();
                unsigned long long wbase = s_run;
                for (int w = 0; w < warp; ++w)
                        wbase += s_w[w];
                if (i < n)
                        out[i] = wbase + x - v;
                __syncthreads();
                if (threadIdx.x == 255)
                        s_run = wbase + x;
                __syncthreads();
        }
}


// varbyte(delta << 1 | changed) [size] payload of one hit with a payload (PAYLOADS): its bytes, and the bytes themselves at h
__device__ __forceinline__ uint32_t enc_payload_hit_len(uint32_t delta, uint32_t len, uint32_t prev_len) {
        const uint32_t ch = len != prev_len;
        return vb_len_of((delta << 1) | ch) + ch + len;
}
__device__ __forceinline__ uint8_t *enc_payload_hit_store(uint8_t *h, uint32_t delta, uint32_t len, uint32_t prev_len, unsigned long long v) {
        const uint32_t ch = len != prev_len;
        h                 = vb_store(h, (delta << 1) | ch);
        if (ch)
                *h++ = uint8_t(len);
        for (uint32_t b = 0; b < len; ++b)
                *h++ = uint8_t(v >> (8u * b));
        return h;
}

// size (WRITE = false) or bytes (WRITE = true) of one block, one warp per block.  Up to 128 documents per block (4 lane groups).
// PAYLOADS: every hit carries plens[] / payloads[] (positions are given); a position-0 hit is legal when it has a payload.
template <bool WRITE, bool PAYLOADS = false>
__global__ void __launch_bounds__(128) k_enc_google_blocks(std::conditional_t<PAYLOADS, EncPayloadParams, EncParams> E) {
        const uint64_t g    = uint64_t(blockIdx.x) * 4u + (threadIdx.x >> 5);
        const int      lane = threadIdx.x & 31;
        if (g >= E.nblocks)
                return;
        uint32_t t;
        if (!WRITE) { // the block's term: last term whose first block is <= g (terms without documents have no block)
                uint32_t lo = 0, hi = E.nterms - 1u;
                while (lo < hi) {
                        const uint32_t mid = (lo + hi + 1u) >> 1;
                        if (E.blk_begin[mid] <= g)
                                lo = mid;
                        else
                                hi = mid - 1u;
                }
                t = lo;
                if (lane == 0)
                        E.bterm[g] = t;
        } else
                t = E.bterm[g];
        const uint64_t tb = E.term_begin[t], te = E.term_begin[t + 1];
        const uint64_t j  = g - E.blk_begin[t];
        const uint64_t d0 = tb + j * E.block_docs;
        const uint32_t n  = uint32_t(min(uint64_t(E.block_docs), te - d0));
        const uint32_t prevLast = j ? E.docids[d0 - 1] : 0u, last = E.docids[d0 + n - 1u];
        // pass 1: per-document code lengths (registers), totals
        uint32_t lenD[4], lenF[4], lenH[4], doc[4], fr[4], dl[4];
        uint32_t totD{0}, totF{0}, totH{0};
        bool     bad = false;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                lenD[q] = lenF[q] = lenH[q] = 0;
                doc[q] = fr[q] = dl[q] = 0;
                if (i < n) {
                        const uint32_t d = E.docids[d0 + i], p = (d0 + i) == tb ? 0u : E.docids[d0 + i - 1];
                        bad |= d == 0u || d <= p;
                        doc[q]  = d;
                        dl[q]   = d - p;
                        fr[q]   = E.freqs[d0 + i];
                        lenD[q] = i + 1u < n ? vb_len_of(dl[q]) : 0u; // the last document is implied by the header
                        lenF[q] = vb_len_of(fr[q]);
                        if constexpr (PAYLOADS) {
                                const uint64_t hb = E.hit_begin[d0 + i];
                                uint32_t       pp{0}, pl{0}, h{0};
                                for (uint32_t k = 0; k < fr[q]; ++k) {
                                        const uint32_t pos = E.positions[hb + k], len = E.pay.plens[hb + k];
                                        bad |= (pos == 0u && len == 0u) || pos < pp || pos >= (1u << 14) || len > 8u; // google_codec.cpp:42-49
                                        h += enc_payload_hit_len(pos - pp, len, pl);
                                        pp = pos;
                                        pl = len;
                                }
                                lenH[q] = h;
                        } else if (E.positions) {
                                const uint64_t hb = E.hit_begin[d0 + i];
                                uint32_t       pp{0}, h{0};
                                for (uint32_t k = 0; k < fr[q]; ++k) {
                                        const uint32_t pos = E.positions[hb + k];
                                        bad |= pos == 0u || pos < pp || pos >= (1u << 14); // Limits::MaxPosition (trinity_limits.h:15; google_codec.cpp:47-49)
                                        h += vb_len_of((pos - pp) << 1);
                                        pp = pos;
                                }
                                lenH[q] = h;
                        } else
                                lenH[q] = fr[q]; // positions 1..freq: every delta is 1 -> one byte 0x02
                }
                uint32_t a = lenD[q], b = lenF[q], c = lenH[q];
                for (int o = 16; o; o >>= 1) {
                        a += __shfl_xor_sync(0xffffffffu, a, o);
                        b += __shfl_xor_sync(0xffffffffu, b, o);
                        c += __shfl_xor_sync(0xffffffffu, c, o);
                }
                totD += a;
                totF += b;
                totH += c;
        }
        if (__any_sync(0xffffffffu, bad)) {
                if (lane == 0)
                        atomicExch(E.error, 1u);
                if (!WRITE && lane == 0)
                        E.bsz[g] = 0;
                return;
        }
        const uint32_t blockLength = totD + totF + totH;
        const uint32_t hdr         = vb_len_of(last - prevLast) + vb_len_of(blockLength) + 1u;
        if (!WRITE) {
                if (lane == 0)
                        E.bsz[g] = hdr + blockLength;
                return;
        }
        const uint64_t chunk  = E.term_off[t];
        const uint64_t b0     = E.blk_begin[t];
        const uint64_t blkOff = 2u + (E.boff[g] - E.boff[b0]); // == out.size() - curTermOffset when the block is committed
        uint8_t *      o      = E.out + chunk + blkOff;
        const uint64_t nb     = E.blk_begin[t + 1] - b0;
        const uint32_t step   = E.skiplist_step;
        const uint32_t phase  = uint32_t((uint64_t(E.phase0) + b0) % step);
        if (lane == 0) {
                uint8_t *p = vb_store(o, last - prevLast);
                p          = vb_store(p, blockLength);
                *p         = uint8_t(n);
                const uint64_t c = uint64_t(phase) + j + 1u; // the countdown reaches 0 when c is a multiple of the step
                if (c % step == 0u) {
                        const uint64_t e = c / step - 1u;
                        if (e < 65535u) {
                                const uint64_t blocksBytes = E.boff[b0 + nb] - E.boff[b0];
                                uint8_t *      s           = E.out + chunk + 2u + blocksBytes + e * 8u;
                                const uint32_t off32       = uint32_t(blkOff);
                                s[0] = uint8_t(prevLast), s[1] = uint8_t(prevLast >> 8), s[2] = uint8_t(prevLast >> 16), s[3] = uint8_t(prevLast >> 24);
                                s[4] = uint8_t(off32), s[5] = uint8_t(off32 >> 8), s[6] = uint8_t(off32 >> 16), s[7] = uint8_t(off32 >> 24);
                        }
                }
                if (j == 0) {
                        const uint32_t entries = uint32_t(min(uint64_t(65535u), (uint64_t(phase) + nb) / step));
                        E.out[chunk]           = uint8_t(entries);
                        E.out[chunk + 1]       = uint8_t(entries >> 8);
                }
        }
        // pass 2: every lane writes its documents' codes at the exclusive prefix of the lengths
        uint32_t runD{0}, runF{0}, runH{0};
        uint8_t *pD = o + hdr, *pF = o + hdr + totD, *pH = o + hdr + totD + totF;
#pragma unroll
        for (int q = 0; q < 4; ++q) {
                const uint32_t i = uint32_t(q) * 32u + uint32_t(lane);
                if (uint32_t(q) * 32u >= n)
                        break;
                uint32_t a = lenD[q], b = lenF[q], c = lenH[q];
                for (int s = 1; s < 32; s <<= 1) {
                        const uint32_t ya = __shfl_up_sync(0xffffffffu, a, s), yb = __shfl_up_sync(0xffffffffu, b, s), yc = __shfl_up_sync(0xffffffffu, c, s);
                        if (lane >= s)
                                a += ya, b += yb, c += yc;
                }
                if (i < n) {
                        if (lenD[q])
                                vb_store(pD + runD + a - lenD[q], dl[q]);
                        vb_store(pF + runF + b - lenF[q], fr[q]);
                        uint8_t *h = pH + runH + c - lenH[q];
                        if constexpr (PAYLOADS) {
                                const uint64_t hb = E.hit_begin[d0 + i];
                                uint32_t       pp{0}, pl{0};
                                for (uint32_t k = 0; k < fr[q]; ++k) {
                                        const uint32_t pos = E.positions[hb + k], len = E.pay.plens[hb + k];
                                        h                  = enc_payload_hit_store(h, pos - pp, len, pl, E.pay.payloads[hb + k]);
                                        pp                 = pos;
                                        pl                 = len;
                                }
                        } else if (E.positions) {
                                const uint64_t hb = E.hit_begin[d0 + i];
                                uint32_t       pp{0};
                                for (uint32_t k = 0; k < fr[q]; ++k) {
                                        const uint32_t pos = E.positions[hb + k];
                                        h                  = vb_store(h, (pos - pp) << 1);
                                        pp                 = pos;
                                }
                        } else
                                for (uint32_t k = 0; k < fr[q]; ++k)
                                        h[k] = 0x02u;
                }
                runD += __shfl_sync(0xffffffffu, a, 31);
                runF += __shfl_sync(0xffffffffu, b, 31);
                runH += __shfl_sync(0xffffffffu, c, 31);
        }
}

// bytes of every term's chunk: u16 + blocks + skiplist entries
__global__ void __launch_bounds__(256) k_enc_term_sizes(EncParams E, unsigned long long *chunk_bytes) {
        const uint32_t t = blockIdx.x * 256u + threadIdx.x;
        if (t >= E.nterms)
                return;
        const uint64_t b0 = E.blk_begin[t], nb = E.blk_begin[t + 1] - b0;
        const uint32_t phase = uint32_t((uint64_t(E.phase0) + b0) % E.skiplist_step);
        const uint64_t entries = min(uint64_t(65535u), (uint64_t(phase) + nb) / E.skiplist_step);
        chunk_bytes[t]         = 2u + (E.boff[b0 + nb] - E.boff[b0]) + 8u * entries;
}

cudaError_t launch_enc_term_sizes(const EncParams &E, unsigned long long *chunk_bytes, cudaStream_t stream) {
        if (!E.nterms)
                return cudaSuccess;
        k_enc_term_sizes<<<(E.nterms + 255u) / 256u, 256, 0, stream>>>(E, chunk_bytes);
        return cudaGetLastError();
}

cudaError_t launch_enc_scan(const uint32_t *in, uint64_t n, unsigned long long *partials /* n / 4096 + 2 */, unsigned long long *out /* n + 1 */, cudaStream_t stream) {
        const uint32_t nparts = uint32_t((n + kEncScanSpan - 1) / kEncScanSpan);
        if (!nparts) {
                return cudaMemsetAsync(out, 0, 8, stream);
        }
        k_enc_scan_partials<<<nparts, 256, 0, stream>>>(in, n, partials);
        k_enc_scan_top<<<1, 1024, 0, stream>>>(partials, nparts);
        k_enc_scan_final<<<nparts, 256, 0, stream>>>(in, n, partials, nparts, out);
        return cudaGetLastError();
}

// pay.plens set: the payload instantiation (the hits without payloads keep theirs)
cudaError_t launch_enc_google_sizes(const EncParams &E, const EncPayloads &pay, cudaStream_t stream) {
        if (!E.nblocks)
                return cudaSuccess;
        if (pay.plens)
                k_enc_google_blocks<false, true><<<unsigned((E.nblocks + 3) / 4), 128, 0, stream>>>(EncPayloadParams{E, pay});
        else
                k_enc_google_blocks<false><<<unsigned((E.nblocks + 3) / 4), 128, 0, stream>>>(E);
        return cudaGetLastError();
}
cudaError_t launch_enc_google_write(const EncParams &E, const EncPayloads &pay, cudaStream_t stream) {
        if (!E.nblocks)
                return cudaSuccess;
        if (pay.plens)
                k_enc_google_blocks<true, true><<<unsigned((E.nblocks + 3) / 4), 128, 0, stream>>>(EncPayloadParams{E, pay});
        else
                k_enc_google_blocks<true><<<unsigned((E.nblocks + 3) / 4), 128, 0, stream>>>(E);
        return cudaGetLastError();
}
