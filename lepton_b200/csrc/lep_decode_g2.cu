// lep_decode_g2.cu -- sm_90a decode kernel, second cut of the group design (lep_decode_group.cu): G lanes per Lepton
// thread-segment, 32/G segments per warp in lock step, with the step loop stripped down:
//
//   * the two kinds of counts (6-bit 7x7 non-zero count, 3-bit edge counts; decoder.cc:175-184, 43-62) are fixed-length
//     loops that every live group runs together -- no state, no votes;
//   * the coefficient loops (7x7, horizontal edge, vertical edge, DC) carry a three/four-state machine (exponent / sign /
//     threshold bits / residual bits; decoder.cc:212-240, 257-300) whose per-coefficient set-up only combines tables the
//     lane-parallel phases prepared: exponent offsets per zig-zag position (prior bit length folded in), packed edge
//     contexts (Lakhani prior -> bsr, sign class, threshold context), per-component table bases by remaining count;
//   * end-of-block positions (eob_x / eob_y) are found by the lanes after the 7x7 loop instead of per decision, the
//     residual / threshold table addresses are formed only when a coefficient turns out to need them;
//   * the count trees are read as whole rows before their first bit, so no bit of a count waits for a load;
//   * the stream window is topped up from a word fetched one refill ahead.
//
// Same job descriptors, model layout, work queue and results as lep_decode_group.cu.
#include "lep_common.cuh"
#include "lep_predict.cuh"

namespace lepb200 {

struct G2Bool {                           // vpx_reader (boolreader.hh:184-258), identical in the G lanes of a group
    unsigned long long value;             // stream bits, left aligned
    uint32_t range;
    int valid;                            // bits of `value` that come from the stream (the rest are zero)
    uint32_t next;                        // the next 32-bit word of the stream (big-endian order restored), already loaded
    const uint8_t* p;                     // address `next` was loaded from
    const uint8_t* end;
};

__device__ __forceinline__ uint32_t g2_load_word(const uint8_t* p, const uint8_t* end) {
    uint32_t w = 0;
    const long long rem = end - p;
    if (rem > 0) {
        w = __byte_perm(__ldg(reinterpret_cast<const uint32_t*>(p)), 0u, 0x0123u);
        if (rem < 4) w &= 0xffffffffu << (8 * (4 - (int)rem));        // the padding behind a stream is readable but not zero
    }
    return w;
}
// vpx_reader_fill restated: one aligned big-endian 32-bit word whenever fewer than 32 bits are left; the word after it is
// requested right away so that its latency is hidden behind the next ~40 decisions
__device__ __forceinline__ void g2_refill(G2Bool& r) {
    r.value |= (unsigned long long)r.next << (32 - r.valid);
    r.valid += 32;
    r.p += 4;
    r.next = g2_load_word(r.p, r.end);
}
__device__ __forceinline__ void g2_init(G2Bool& r, const uint8_t* p, uint32_t len) {
    r.value = 0; r.valid = 0; r.range = 255;
    r.p = p; r.end = p + len;
    r.next = g2_load_word(r.p, r.end);
    g2_refill(r);
    // marker bit at p = 128 (boolreader.cc:26-35); no model involved
    const uint32_t split = (r.range * 128u + 128u) >> 8;
    const uint32_t bit = (uint32_t)(r.value >> 56) >= split;
    const uint32_t range = bit ? r.range - split : split;
    if (bit) r.value -= (unsigned long long)split << 56;
    const int shift = __clz(range) - 24;
    r.range = range << shift; r.value <<= shift; r.valid -= shift;
}

// VPXBoolReader::get (vpx_bool_reader.hh:45-57) = vpx_read + Branch::record_obs_and_update, in three pieces so that the
// step loops can put the NEXT decision's model load between the bit and the bookkeeping:
//   g2_bit         the decision itself: probability of the branch word, split, window top-up, compare   (on the serial chain)
//   g2_update      range / window renormalisation                                                      (off the chain)
//   g2_model_word  the branch word after the observation                                                (off the chain)
__device__ __forceinline__ uint32_t g2_bit(G2Bool& r, const uint32_t* rcp, uint32_t w, uint32_t& split) {
    const uint32_t prob = branch_prob(w, rcp);
    split = (r.range * prob + (256 - prob)) >> 8;
    if (r.valid < 32) g2_refill(r);
    return (uint32_t)(r.value >> 56) >= split;                     // value >= split << 56  <=>  top byte >= split
}
__device__ __forceinline__ void g2_update(G2Bool& r, uint32_t split, uint32_t bit) {
    const uint32_t range = bit ? r.range - split : split;
    if (bit) r.value -= (unsigned long long)split << 56;
    const int shift = __clz(range) - 24;
    r.range = range << shift;
    r.value <<= shift;
    r.valid -= shift;
}
__device__ __forceinline__ uint32_t g2_model_word(uint32_t w, uint32_t bit) {
    const bool plain = (w & 0xffu) < 254u && (w >> 8) < 254u;       // no count about to saturate, not the special state
    return (plain ? w + (bit ? 0x100u : 1u) : branch_update(w, bit)) & 0xffffu;
}
// one whole decision where nothing is pipelined (fixed-length count loops use the pieces directly)
__device__ __forceinline__ uint32_t g2_get(G2Bool& r, uint16_t* model, const uint32_t* rcp, uint32_t addr, uint32_t w) {
    uint32_t split;
    const uint32_t bit = g2_bit(r, rcp, w, split);
    g2_update(r, split, bit);
    model[addr] = (uint16_t)g2_model_word(w, bit);                 // all lanes of the group store the same value
    return bit;
}
#ifdef LEPB200_EMU
#define G2_EMU_BARRIER() __syncwarp()      // CPU warp emulator only: lanes run one after the other there, so the lanes of a group must
                                           // all have read a branch word before the first of them writes it back (fixed-length count loops;
                                           // the coefficient loops vote once per decision, which orders them the same way)
#else
#define G2_EMU_BARRIER()
#endif

// Branch words of the fixed-length count trees are read as whole rows (a tree level's candidates are contiguous), so
// that no bit of a count waits for a load the previous bit chose: halfword i of 8 packed in a uint4, of 4 in a uint2.
__device__ __forceinline__ uint32_t g2_half8(uint4 v, uint32_t i) {
    const uint32_t u = (i & 4u) ? ((i & 2u) ? v.w : v.z) : ((i & 2u) ? v.y : v.x);
    return (u >> ((i & 1u) << 4)) & 0xffffu;
}
__device__ __forceinline__ uint32_t g2_half4(uint2 v, uint32_t i) {
    return (((i & 2u) ? v.y : v.x) >> ((i & 1u) << 4)) & 0xffffu;
}
// the 7x7 count tree (m_nz7): rows 5..2 hold 1, 2, 4, 8 words at the row start and do not depend on a bit of the count,
// so they are requested together, as early as the tree's base is known
struct G2NzTop { uint32_t r5, r4; uint2 r3; uint4 r2; };
__device__ __forceinline__ G2NzTop g2_nz_top(const uint16_t* t) {
    G2NzTop v;
    v.r5 = t[5 << 5];
    v.r4 = *reinterpret_cast<const uint32_t*>(t + (4 << 5));
    v.r3 = *reinterpret_cast<const uint2*>(t + (3 << 5));
    v.r2 = *reinterpret_cast<const uint4*>(t + (2 << 5));
    return v;
}
// an edge count tree (m_nze): rows 2, 1, 0 of 1, 2, 4 words, 24 bytes in all
struct G2EdgeTree { uint32_t r2, r1; uint2 r0; };
__device__ __forceinline__ G2EdgeTree g2_edge_tree(const uint16_t* t) {
    G2EdgeTree v;
    v.r2 = t[2 << 2];
    v.r1 = *reinterpret_cast<const uint32_t*>(t + (1 << 2));
    v.r0 = *reinterpret_cast<const uint2*>(t);
    return v;
}

enum : int { G2_EXP = 0, G2_SIGN = 1, G2_THR = 2, G2_RES = 3 };

// shared memory of one group
struct alignas(16) G2GroupSmem {
    int16_t blk[4][64];                   // raster order: [0],[1] current / left (ping-pong); [2],[3] above / above-left (ping-pong)
    int32_t tmp[64];                      // IDCT intermediate; before the IDCT: tmp[0..24] = exponent offsets of the 49 inner positions
                                          // (uint16 each), tmp[32..45] = packed contexts of the 14 edge coefficients
    int16_t pix[64];                      // pixels of the block without its DC
    int16_t ledge[8];                     // right-column edge prediction of the left neighbour (block_context.hh:44-78)
};
static_assert(sizeof(G2GroupSmem) == 512 + 256 + 128 + 16, "group scratch layout");

template <int G> struct G2Cfg {
    static constexpr int S = 32 / G;                                               // groups (thread-segments) per warp
    static constexpr int WARPS = (G >= 4) ? 4 : G;                                 // static shared memory stays under 48 KB
    static constexpr int THREADS = WARPS * 32;
};

template <int G> __device__ __forceinline__ int g2_sum(int v) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) v += __shfl_xor_sync(FULL, v, d);
    return v;
}
template <int G> __device__ __forceinline__ int g2_min(int v) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) v = min(v, __shfl_xor_sync(FULL, v, d));
    return v;
}
template <int G> __device__ __forceinline__ int g2_max(int v) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) v = max(v, __shfl_xor_sync(FULL, v, d));
    return v;
}
template <int G> __device__ __forceinline__ uint32_t g2_or(uint32_t v) {
#pragma unroll
    for (int d = 1; d < G; d <<= 1) v |= __shfl_xor_sync(FULL, v, d);
    return v;
}

// packed context of one edge coefficient, prepared by the lanes from its Lakhani prediction (model.hh:405-440,1100-1122):
//   bits 0-3 bsr = bit length of min(|prior|, 1023), 4-5 sign class of the prior (0 zero, 1 positive, 2 negative),
//   6-8 min_threshold of the position, 9-16 threshold context min(|prior| >> min_threshold, 255)
__device__ __forceinline__ uint32_t g2_edge_info(int prior, int min_thr) {
    const int bsr = bitlen((uint32_t)min(iabs(prior), 1023));
    const int p16 = (int)(int16_t)prior;
    const int sctx = p16 == 0 ? 0 : (p16 > 0 ? 1 : 2);
    const int ctx_abs = iabs(prior) & 0xffff;
    return (uint32_t)bsr | ((uint32_t)sctx << 4) | ((uint32_t)min_thr << 6) | ((uint32_t)min(ctx_abs >> min_thr, 255) << 9);
}

template <int G>
__global__ void __launch_bounds__(G2Cfg<G>::THREADS)
lep_decode_g2_kernel(const ImageDesc* __restrict__ images, SegDesc* __restrict__ segs, int first, int count, const int* __restrict__ order,
                     int* __restrict__ work_counter, uint16_t* __restrict__ model_pool, uint8_t* __restrict__ row_pool, size_t row_pool_stride) {
    constexpr int S = G2Cfg<G>::S;
    constexpr int CPL = 64 / G;           // coefficients of a block per lane (aligned order)
    __shared__ uint32_t s_rcp[512];
    __shared__ uint8_t s_a2r[64];         // aligned index -> raster index
    __shared__ uint8_t s_nzbin[64];       // remaining non-zero count -> bin (jpeg_meta.hh:72-170 row 9)
    __shared__ uint32_t s_eb[2][52];      // [ci][remaining count]: base of the 7x7 exponent table slice of that bin
    __shared__ G2GroupSmem s_grp[G2Cfg<G>::WARPS * S];
    for (int i = threadIdx.x; i < 512; i += blockDim.x) s_rcp[i] = i < 2 ? 0u : (uint32_t)((0x100000000ull + i - 1) / i);
    for (int i = threadIdx.x; i < 64; i += blockDim.x) { s_a2r[i] = c_aligned_to_raster[i]; s_nzbin[i] = i < 50 ? c_nonzero_to_bin[i] : 0; }
    for (int i = threadIdx.x; i < 2 * 52; i += blockDim.x) {
        const int cc = i / 52, n = i % 52;
        s_eb[cc][n] = m_exp7(cc, n < 50 ? c_nonzero_to_bin[n] : 0, 0, 0);
    }
    __syncthreads();
    const int lane = lane_id();
    const int sub = lane & (G - 1);                       // this lane's place in its group
    const int gbase = lane & ~(G - 1);                    // first lane of the group
    const int slot = (blockIdx.x * G2Cfg<G>::WARPS + (threadIdx.x >> 5)) * S + lane / G;       // row buffer of this group
    G2GroupSmem& gs = s_grp[(threadIdx.x >> 5) * S + lane / G];
    uint16_t* const eoff = reinterpret_cast<uint16_t*>(gs.tmp);          // 7x7: (zz * 12 + bsr) << 4
    uint32_t* const einfo = reinterpret_cast<uint32_t*>(gs.tmp) + 32;    // edges: g2_edge_info
    uint8_t* rowbuf = row_pool + (size_t)slot * row_pool_stride;

    // ---- segment state (identical in the lanes of a group)
    bool alive = false;                   // a segment is in progress
    bool exhausted = false;               // the queue is empty: this group is done
    SegDesc* sdp = nullptr;
    const ImageDesc* gp = images;
    uint16_t* model = model_pool;
    int seg_min_y = 0, seg_max_y = 0;
    bool seg_last = false;
    G2Bool br;
    br.value = 0; br.valid = 0; br.range = 255; br.next = 0; br.p = nullptr; br.end = nullptr;
    unsigned long long ndec = 0;
    uint32_t top_mask = 7u, index = 0;
    int bw0 = 0, bw1 = 0, bw2 = 0, nzs0 = 0, nzs1 = 0;
    size_t nz_base = 0;
    // ---- row / block cursor (row iteration of lepton_codec.hh:41-100)
    int c = 0, ci = 0, y = 0, w = 0, x = 0, q0 = 1, pc = 0, pa = 2, nz_left = 0;
    bool has_above = false, need_row = true;
    int16_t* rowp = nullptr;
    const int16_t* abovep = nullptr;
    const uint16_t* q = nullptr;
    int16_t* redge = nullptr;
    uint8_t* rnz = nullptr;
    const int32_t* icx = nullptr;
    const int32_t* icy = nullptr;
    const uint8_t* mthr = nullptr;
    // ---- the 7x7 count tree of the block to come: base and top rows, requested at the end of the previous block of the
    //      row when it has one (in flight during phases (1) and (1b)), else in (1b)
    uint32_t cnt_addr = 0;
    G2NzTop nzt = {};
    bool cnt_ready = false;

    for (;;) {
        // ---- (0a) a free group takes the next segment of the queue
        const bool want_job = !alive && !exhausted;
        if (__any_sync(FULL, want_job)) {
            int job = -1;
            if (want_job && sub == 0) job = atomicAdd(work_counter, 1);
            job = __shfl_sync(FULL, job, gbase);
            if (want_job) {
                if (job >= count) {
                    exhausted = true;
                } else {
                    const int sidx = order[first + job];
                    sdp = &segs[sidx];
                    if (sdp->status == ST_OK) {               // else rejected on the host (e.g. zero quantiser, model.hh:257-262)
                        gp = &images[sdp->image];
                        model = model_pool + (size_t)job * M_TOTAL;          // zero-filled before the launch
                        seg_min_y = sdp->min_y; seg_max_y = sdp->max_y; seg_last = sdp->is_last != 0;
                        g2_init(br, reinterpret_cast<const uint8_t*>(sdp->stream), sdp->cap);
                        ndec = 0; top_mask = 7u; index = 0;
                        bw0 = gp->bch[0]; bw1 = gp->ncmp > 1 ? gp->bch[1] : 0; bw2 = gp->ncmp > 2 ? gp->bch[2] : 0;
                        nz_base = (size_t)(bw0 + bw1 + bw2) * 16;
                        nzs0 = (bw0 + 15) & ~15; nzs1 = (bw1 + 15) & ~15;
                        need_row = true;
                        alive = true;
                    }
                }
            }
        }
        // ---- (0b) move to the next row when the previous one is finished (per group, once per row)
        if (alive && need_row) {
            const ImageDesc& g = *gp;
            for (;;) {
                const RowSpec rs = row_spec_from_index(index++, g);
                if (rs.done || (rs.luma_y >= seg_max_y && !seg_last)) { alive = false; break; }
                if (rs.skip || rs.luma_y < seg_min_y) continue;
                c = rs.component; y = rs.curr_y;
                has_above = !((top_mask >> c) & 1u);
                top_mask &= ~(1u << c);
                ci = c == 0 ? 0 : 1;
                w = g.bch[c];
                rowp = reinterpret_cast<int16_t*>(g.plane[c]) + (size_t)y * w * 64;
                abovep = rowp - (size_t)w * 64;
                q = g.q[c];
                q0 = q[0];
                redge = reinterpret_cast<int16_t*>(rowbuf + (size_t)(c == 0 ? 0 : (c == 1 ? bw0 : bw0 + bw1)) * 16);
                rnz = rowbuf + nz_base + (c == 0 ? 0 : (c == 1 ? nzs0 : nzs0 + nzs1));
                icx = g.icos_x[c];
                icy = g.icos_y[c];
                mthr = g.min_thr[c];
                x = 0; pc = 0; pa = 2; nz_left = 0;
                need_row = false;
                break;
            }
            if (!alive && sub == 0) {                         // the segment is complete
                sdp->status = ST_OK;
                sdp->len = (uint32_t)(br.p - reinterpret_cast<const uint8_t*>(sdp->stream));       // whole words
                sdp->ndecisions_lo = (uint32_t)ndec;
                sdp->ndecisions_hi = (uint32_t)(ndec >> 32);
            }
        }
        if (__all_sync(FULL, exhausted)) break;
        // a group that just finished its segment sits this block round out and takes the next segment at the top

        const bool has_left = x > 0;
        int16_t* rcur = gs.blk[pc];
        const int16_t* rleft = gs.blk[pc ^ 1];
        int16_t* rabove = gs.blk[pa];
        const int16_t* raleft = gs.blk[pa ^ 1];
        uint32_t nd = 0;                  // decisions of this block
        int nz = 0;

        // ---- (1) above block -> raster copy, clear the current block
        if (alive) {
            if (has_above) {
                const uint32_t* src = reinterpret_cast<const uint32_t*>(abovep + (size_t)x * 64) + sub * (CPL / 2);
#pragma unroll
                for (int k = 0; k < CPL / 2; ++k) {
                    const uint32_t u = src[k];
                    const int a = sub * CPL + 2 * k;
                    rabove[s_a2r[a]] = (int16_t)(u & 0xffff);
                    rabove[s_a2r[a + 1]] = (int16_t)(u >> 16);
                }
            }
#pragma unroll
            for (int k = 0; k < CPL / 2; ++k) reinterpret_cast<uint32_t*>(rcur)[sub * (CPL / 2) + k] = 0u;
        }
        __syncwarp();
        // ---- (1b) exponent offsets of the 49 inner positions: compute_aavrg (model.hh:895-924) -> bit length -> (zz*12+bsr)<<4
        if (alive) {
            for (int zz = sub; zz < 49; zz += G) {
                const int coord = s_a2r[zz];
                uint32_t pr = 0;
                if (has_left && has_above) {
                    const uint32_t L = (uint32_t)iabs(rleft[coord]) & 0xffff, A = (uint32_t)iabs(rabove[coord]) & 0xffff;
                    pr = (((L + A) * 13u + (((uint32_t)iabs(raleft[coord]) & 0xffff) * 6u)) & 0xffff) >> 5;
                } else if (has_left || has_above) {
                    const int16_t nb = has_left ? rleft[coord] : rabove[coord];
                    pr = (uint32_t)iabs((int)(int16_t)((uint32_t)iabs(nb) & 0xffff));
                }
                eoff[zz] = (uint16_t)((zz * 12 + bitlen(min(pr, 1023u))) << 4);
            }
            if (!cnt_ready) {
                const int nz_above = has_above ? (int)rnz[x] : 0;
                int ctx = 0;
                if (has_above && !has_left) ctx = (nz_above + 1) / 2;
                else if (has_left && !has_above) ctx = (nz_left + 1) / 2;
                else if (has_left && has_above) ctx = (nz_above + nz_left + 2) / 4;
                cnt_addr = m_nz7(ci, s_nzbin[ctx], 0, 0);
                nzt = g2_nz_top(model + cnt_addr);
            }
        }
        cnt_ready = false;
        __syncwarp();

        // ---- (2a) the 7x7 non-zero count: six decisions, every live group in step (decoder.cc:175-184).  Level idx of the
        //      tree is the row cnt_addr + idx * 32, indexed by the bits above it.  Rows 5..2 are in registers already; the
        //      8 words of row 1 that the first bit leaves possible, and of row 0 after the second bit, are requested three
        //      decisions before they are used.  No word of the tree is read twice, so nothing needs forwarding.
        {
            uint4 r1 = make_uint4(0u, 0u, 0u, 0u), r0 = r1;
            uint32_t prefix = 0;
#pragma unroll
            for (int idx = 5; idx >= 0; --idx) {
                const uint32_t mw = idx == 5 ? nzt.r5 : idx == 4 ? (nzt.r4 >> (prefix << 4)) & 0xffffu
                                  : idx == 3 ? g2_half4(nzt.r3, prefix) : idx == 2 ? g2_half8(nzt.r2, prefix)
                                  : idx == 1 ? g2_half8(r1, prefix & 7u) : g2_half8(r0, prefix & 7u);
                uint32_t split = 0, bit = 0;
                if (alive) bit = g2_bit(br, s_rcp, mw, split);
                const uint32_t p1 = (prefix << 1) | bit;
                if (alive && idx == 5) r1 = *reinterpret_cast<const uint4*>(model + cnt_addr + (1u << 5) + (p1 << 3));
                if (alive && idx == 4) r0 = *reinterpret_cast<const uint4*>(model + cnt_addr + (p1 << 3));
                if (idx >= 4) G2_EMU_BARRIER();
                if (alive) {
                    model[cnt_addr + ((uint32_t)idx << 5) + prefix] = (uint16_t)g2_model_word(mw, bit);
                    g2_update(br, split, bit);
                    prefix = p1;
                }
            }
            nz = (int)prefix;
            if (alive) nd += 6;
        }
        bool bad = false;                 // a stream that announces more than 49 coefficients ends its segment (decoder.cc:182-184)
        if (alive && nz > 49) { bad = true; alive = false; }

        // ---- (2b) the 7x7 coefficients in zig-zag order (== aligned order 0..48) until the announced count is used up.
        //      One decision per live group and round.  What sits on the serial chain of a group is only: branch word ->
        //      probability -> split -> compare -> SELECT of the next branch address -> load.  The two candidate addresses
        //      (next decision if this bit is 0 / if it is 1) are prepared from the grammar state BEFORE the bit is known,
        //      in the shadow of the previous load, together with the write-back, the window update and the state update
        //      (straight-line code: groups in different states share every instruction).  Consecutive decisions never use
        //      the same branch, except for the saturated threshold index of the edge loop; the forwarding line covers it.
        {
            int zz = 0, left_nz = nz, st = G2_EXP, len = 0, ri = 0, val = 0;
            bool neg = false;
            uint32_t addr = 0, a0 = 0, a1 = 0;
            bool busy = alive && nz > 0, b0 = busy, b1 = busy;
            const uint32_t sign_addr = m_sign(ci, 0, 0);
            if (busy) {
                const uint32_t eb = s_eb[ci][left_nz];
                addr = eb + eoff[0];
                a1 = addr + 1; a0 = eb + eoff[1];          // after the first exponent bit of position 0
            }
            uint32_t mw = busy ? model[addr] : 0u;
            while (__any_sync(FULL, busy)) {
                if (busy) {
                    // ---- on the chain
                    uint32_t split;
                    const uint32_t bit = g2_bit(br, s_rcp, mw, split);
                    const uint32_t naddr = bit ? a1 : a0;
                    const bool nbusy = bit ? b1 : b0;
                    uint32_t mwn = nbusy ? model[naddr] : 0u;
                    // ---- in the shadow of that load: write-back, window, grammar state, decoded value
                    const uint32_t neww = g2_model_word(mw, bit);
                    model[addr] = (uint16_t)neww;                  // all lanes of the group store the same value
                    if (naddr == addr) mwn = neww;
                    g2_update(br, split, bit);
                    ++nd;
                    const int isE = st == G2_EXP, isS = st == G2_SIGN, isR = st == G2_RES;
                    const int cont = isE & (int)bit & (int)(len < 10);               // exponent goes on
                    const int len1 = len + (isE & (int)bit);
                    const int ev0 = isE & (cont ^ 1) & (int)(len1 == 0);              // zero coefficient
                    const int toS = isE & (cont ^ 1) & (int)(len1 != 0);
                    const int ris = len - 2;                                          // sign state: first residual bit
                    const int evS = isS & (int)(ris < 0), toR = isS & (int)(ris >= 0);
                    const int evR = isR & (int)(ri == 0);
                    const int evN = evS | evR, ev = ev0 | evN;                        // a (non-zero) coefficient is complete
                    const int nval = isS ? (1 << ((len - 1) & 31)) : (isR ? (val | ((int)bit << (ri & 31))) : val);
                    const bool nneg = isS ? !bit : neg;
                    if (evN && sub == 0) rcur[s_a2r[zz]] = (int16_t)(nneg ? -nval : nval);
                    left_nz -= evN; zz += ev;
                    st = toS ? G2_SIGN : toR ? G2_RES : ev ? G2_EXP : st;
                    len = ev ? 0 : len1;
                    ri = isS ? ris : ri - isR;
                    val = nval; neg = nneg; addr = naddr; busy = nbusy; mw = mwn;
                    // ---- candidates of the decision after the one just requested
                    if (busy) {
                        const int zn = min(zz + 1, 48);
                        const bool lastpos = zz == 48;
                        const bool doneN = left_nz == 1 || lastpos;              // after the non-zero coefficient in progress
                        const uint32_t nextN = s_eb[ci][left_nz - 1] + eoff[zn];
                        const bool inE = st == G2_EXP, inS = st == G2_SIGN;
                        const bool fin = inS ? len < 2 : ri == 0;                // the coming decision completes the coefficient
                        const uint32_t cont_a = inS ? m_resn(ci, s_a2r[zz], s_nzbin[left_nz]) + (uint32_t)(len - 2) : addr - 1;
                        const uint32_t common = fin ? nextN : cont_a;
                        const bool commonB = fin ? !doneN : true;
                        a1 = inE ? (len < 10 ? addr + 1 : sign_addr) : common;
                        a0 = inE ? (len == 0 ? s_eb[ci][left_nz] + eoff[zn] : sign_addr) : common;
                        b1 = inE ? true : commonB;
                        b0 = inE ? (len == 0 ? !lastpos : true) : commonB;
                    }
                }
            }
        }
        __syncwarp();

        // ---- (3) eob_x / eob_y of the 7x7 part (encoder.cc:219-255 tracks them per coefficient), then the Lakhani
        //          predictions of the 14 edge coefficients (model.hh:1033-1071) packed into their contexts
        int eobx = 0, eoby = 0;
        {
            uint32_t colmask = 0, rowmask = 0;
            if (alive) {
                for (int r = 1 + sub; r < 8; r += G) {
                    const uint4 u = *reinterpret_cast<const uint4*>(rcur + r * 8);
                    uint32_t m = 0;
                    m |= (u.x >> 16) ? 2u : 0u;
                    m |= (u.y & 0xffffu) ? 4u : 0u;   m |= (u.y >> 16) ? 8u : 0u;
                    m |= (u.z & 0xffffu) ? 16u : 0u;  m |= (u.z >> 16) ? 32u : 0u;
                    m |= (u.w & 0xffffu) ? 64u : 0u;  m |= (u.w >> 16) ? 128u : 0u;
                    colmask |= m;
                    if (m) rowmask |= 1u << r;
                }
            }
            colmask = g2_or<G>(colmask); rowmask = g2_or<G>(rowmask);
            eobx = colmask ? 31 - __clz(colmask) : 0;
            eoby = rowmask ? 31 - __clz(rowmask) : 0;
        }
        G2EdgeTree eth = {}, etv = {};
        if (alive) {
            eth = g2_edge_tree(model + m_nze(0, ci, eobx, (nz + 3) / 7, 0, 0));
            etv = g2_edge_tree(model + m_nze(1, ci, eoby, (nz + 3) / 7, 0, 0));
            for (int k = sub; k < 14; k += G) {
                int p = 0, coord;
                if (k < 7) { coord = k + 1; if (has_above) p = lak_pred(rcur, rabove, icx + (k + 1) * 8, k + 1, 8); }
                else { coord = 8 * (k - 6); if (has_left) p = lak_pred(rcur, rleft, icy + (k - 6) * 8, 8 * (k - 6), 1); }
                einfo[k] = g2_edge_info(p, mthr[coord]);
            }
        }
        __syncwarp();

        // ---- (4) edges: horizontal (raster 1..7) then vertical (raster 8..56): 3-bit count, then coefficients (decoder.cc:43-160)
#pragma unroll 1
        for (int vert = 0; vert < 2; ++vert) {
            int ne = 0;
            {
                // the whole tree was read in (3): level idx is the row base + idx * 4, indexed by the bits above it
                const uint32_t base = m_nze(vert, ci, vert ? eoby : eobx, (nz + 3) / 7, 0, 0);
                const G2EdgeTree t = vert ? etv : eth;
                uint32_t prefix = 0;
#pragma unroll
                for (int idx = 2; idx >= 0; --idx) {
                    const uint32_t mw = idx == 2 ? t.r2 : idx == 1 ? (t.r1 >> (prefix << 4)) & 0xffffu : g2_half4(t.r0, prefix);
                    uint32_t split = 0, bit = 0;
                    if (alive) {
                        bit = g2_bit(br, s_rcp, mw, split);
                        model[base + ((uint32_t)idx << 2) + prefix] = (uint16_t)g2_model_word(mw, bit);
                        g2_update(br, split, bit);
                        prefix = (prefix << 1) | bit;
                    }
                }
                ne = (int)prefix;
                if (alive) nd += 3;
            }
            int ln = 0, st = G2_EXP, len = 0, ri = 0, val = 0;
            bool neg = false;
            uint32_t addr = 0, e = 0, so = 1, thr_base = 0, a0 = 0, a1 = 0;
            const uint32_t expx_base = M_EXPX + (uint32_t)((ci * 8) * 15 * 12 * 16) + (uint32_t)(vert * 7 * 12 * 16);
            const uint32_t sign_base = M_SIGN + (uint32_t)(ci * 48);
            const int cstep = vert ? 8 : 1;                       // raster distance between the coefficients of this edge
            constexpr uint32_t NE_STRIDE = 15 * 12 * 16;          // exponent contexts of one remaining-count value
            bool busy = alive && ne > 0, b0 = busy, b1 = busy;
            if (busy) {
                e = einfo[vert * 7];
                addr = expx_base + (uint32_t)ne * NE_STRIDE + ((e & 15u) << 4);
                a1 = addr + 1;
                a0 = expx_base + (uint32_t)ne * NE_STRIDE + (uint32_t)(12 * 16) + ((einfo[vert * 7 + 1] & 15u) << 4);
            }
            uint32_t mw = busy ? model[addr] : 0u;
            while (__any_sync(FULL, busy)) {
                if (busy) {
                    // ---- on the chain (see the 7x7 loop)
                    uint32_t split;
                    const uint32_t bit = g2_bit(br, s_rcp, mw, split);
                    const uint32_t naddr = bit ? a1 : a0;
                    const bool nbusy = bit ? b1 : b0;
                    uint32_t mwn = nbusy ? model[naddr] : 0u;
                    // ---- in the shadow of that load
                    const uint32_t neww = g2_model_word(mw, bit);
                    model[addr] = (uint16_t)neww;
                    if (naddr == addr) mwn = neww;                 // saturated threshold index: the same branch twice in a row
                    g2_update(br, split, bit);
                    ++nd;
                    const int isE = st == G2_EXP, isS = st == G2_SIGN, isT = st == G2_THR, isR = st == G2_RES;
                    const int cont = isE & (int)bit & (int)(len < 10);
                    const int len1 = len + (isE & (int)bit);
                    const int ev0 = isE & (cont ^ 1) & (int)(len1 == 0);
                    const int toS = isE & (cont ^ 1) & (int)(len1 != 0);
                    const int mt = (int)((e >> 6) & 7u);                              // min_threshold of this position
                    const int ris = len - 2;
                    const int evS = isS & (int)(ris < 0);
                    const int toT = isS & (int)(ris >= 0) & (int)(ris >= mt), toRs = isS & (int)(ris >= 0) & (int)(ris < mt);
                    const int rit = ri - 1;                                           // threshold / residual states: next bit
                    const int evT = isT & (int)(ri == 0), toRt = isT & (int)(ri != 0) & (int)(rit < mt);
                    const int evR = isR & (int)(ri == 0);
                    const int evN = evS | evT | evR, ev = ev0 | evN;
                    const int nval = isS ? (1 << ((len - 1) & 31)) : ((isT | isR) ? (val | ((int)bit << (ri & 31))) : val);
                    const bool nneg = isS ? !bit : neg;
                    if (evN && sub == 0) rcur[(ln + 1) * cstep] = (int16_t)(nneg ? -nval : nval);
                    so = isT ? min((so << 1) | bit, 127u) : 1u;
                    thr_base = isS ? m_thr(ci, (int)((e >> 9) & 255u), min(len - mt, 7)) : thr_base;
                    ne -= evN; ln += ev;
                    if (ev) e = einfo[vert * 7 + min(ln, 6)];
                    st = toS ? G2_SIGN : toT ? G2_THR : (toRs | toRt) ? G2_RES : ev ? G2_EXP : st;
                    len = ev ? 0 : len1;
                    ri = isS ? ris : ri - (isT | isR);
                    val = nval; neg = nneg; addr = naddr; busy = nbusy; mw = mwn;
                    // ---- candidates of the decision after the one just requested
                    if (busy) {
                        const int mt2 = (int)((e >> 6) & 7u);
                        const bool lastpos = ln == 6;
                        const bool doneN = ne == 1 || lastpos;                   // after the non-zero coefficient in progress
                        const uint32_t nxt = (uint32_t)((ln + 1) * (12 * 16)) + ((einfo[vert * 7 + min(ln + 1, 6)] & 15u) << 4);
                        const uint32_t nextN = expx_base + (uint32_t)(ne - 1) * NE_STRIDE + nxt;
                        const uint32_t rb = m_resn(ci, (ln + 1) * cstep, ne);
                        const bool inE = st == G2_EXP, inS = st == G2_SIGN, inT = st == G2_THR;
                        const int r2 = inS ? len - 2 : ri - 1;                   // bit index of the decision after the coming one
                        const bool fin = r2 < 0;                                 // the coming decision completes the coefficient
                        const bool thr = r2 >= mt2 && (inS || inT);              // ... or it is followed by a threshold bit
                        const uint32_t tb = inS ? m_thr(ci, (int)((e >> 9) & 255u), min(len - mt2, 7)) : thr_base;
                        const uint32_t so0 = inS ? 1u : min(so << 1, 127u), so1 = inS ? 1u : min((so << 1) | 1u, 127u);
                        const uint32_t rest = (inS || inT) ? rb + (uint32_t)r2 : addr - 1;        // residual bit after sign / threshold, or the next one down
                        const uint32_t c0 = fin ? nextN : thr ? tb + so0 : rest;
                        const uint32_t c1 = fin ? nextN : thr ? tb + so1 : rest;
                        const bool cb = fin ? !doneN : true;
                        const uint32_t sa = sign_base + ((e >> 4) & 3u) * 12u + (e & 15u);
                        a1 = inE ? (len < 10 ? addr + 1 : sa) : c1;
                        a0 = inE ? (len == 0 ? expx_base + (uint32_t)ne * NE_STRIDE + nxt : sa) : c0;
                        b1 = inE ? true : cb;
                        b0 = inE ? (len == 0 ? !lastpos : true) : cb;
                    }
                }
            }
        }
        __syncwarp();

        // ---- (5) DC: pixels of the block without its DC (8x8 IDCT, rows then columns, G lanes), prediction from the
        //          neighbours' edge pixels
        if (alive) {
            for (int r = sub; r < 8; r += G) {
                int32_t in[8], out[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) in[k] = (int32_t)rcur[r * 8 + k] * (int32_t)q[r * 8 + k];
                if (r == 0) in[0] = 0;
                idct_row(in, out);
#pragma unroll
                for (int k = 0; k < 8; ++k) gs.tmp[r * 8 + k] = out[k];
            }
        }
        __syncwarp();
        if (alive) {
            for (int col = sub; col < 8; col += G) {
                int32_t in[8], out[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) in[k] = gs.tmp[k * 8 + col];
                idct_col(in, out);
#pragma unroll
                for (int k = 0; k < 8; ++k) gs.pix[k * 8 + col] = (int16_t)out[k];
            }
        }
        __syncwarp();
        int pred = 0;
        uint32_t dc_exp = 0, dc_sign = 0, dc_res = 0;
        {
            // adv_predict_dc_pix (model.hh:678-784), 16-bit lane arithmetic of the SSE build; 16 estimates over the G lanes
            int sl = 0, sa = 0, mnl = 32767, mxl = -32768, mna = 32767, mxa = -32768;
            if (alive) {
                for (int i = sub; i < 16; i += G) {
                    if (i < 8) {
                        if (has_left) {
                            const int16_t p0 = gs.pix[i * 8], p1 = gs.pix[i * 8 + 1];
                            const int16_t delta = (int16_t)(p0 - p1);
                            const int est = (int16_t)((int16_t)((int16_t)gs.ledge[i] - half_rz16(delta)) - (int16_t)(p0 + 1024));
                            sl += est; mnl = min(mnl, est); mxl = max(mxl, est);
                        }
                    } else if (has_above) {
                        const int j = i - 8;
                        const int16_t p0 = gs.pix[j], p1 = gs.pix[8 + j];
                        const int16_t delta = (int16_t)(p0 - p1);
                        const int est = (int16_t)((int16_t)((int16_t)redge[(size_t)x * 8 + j] - half_rz16(delta)) - (int16_t)(p0 + 1024));
                        sa += est; mna = min(mna, est); mxa = max(mxa, est);
                    }
                }
            }
            sl = g2_sum<G>(sl); sa = g2_sum<G>(sa);
            mnl = g2_min<G>(mnl); mna = g2_min<G>(mna);
            mxl = g2_max<G>(mxl); mxa = g2_max<G>(mxa);
            if (alive) {
                int avgmed = 0, unc = 0, unc2 = 0;
                if (has_left || has_above) {
                    int a0, a1, mn_all, mx_all;
                    if (has_left && has_above) { a0 = sl; a1 = sa; mn_all = min(mnl, mna); mx_all = max(mxl, mxa); }
                    else if (has_left) { a0 = a1 = sl; mn_all = mnl; mx_all = mxl; }
                    else { a0 = a1 = sa; mn_all = mna; mx_all = mxa; }
                    avgmed = (a0 + a1) >> 1;
                    unc = (mx_all - mn_all) >> 3;
                    a0 -= avgmed; a1 -= avgmed;
                    int far_afield = a1;
                    if (iabs(a0) < iabs(a1)) far_afield = a0;
                    unc2 = far_afield >> 3;
                }
                pred = (div_trunc_small(avgmed, q0) + 4) >> 3;
                const int lm = min(bitlen((uint32_t)iabs(unc) & 0xffff), 11), lo16 = min(bitlen((uint32_t)iabs(unc2) & 0xffff), 16);
                const int sctx = unc2 >= 0 ? (unc2 == 0 ? 3 : 2) : 1;
                dc_exp = m_expdc(lm, lo16); dc_sign = m_sign(ci, 0, sctx); dc_res = m_resdc(lm);
            }
        }

        // ---- (6) the DC coefficient: exponent / sign / residual bits (decoder.cc:286-304), same scheme
        int dcv = 0;
        {
            int st = G2_EXP, len = 0, ri = 0, val = 0;
            bool neg = false;
            uint32_t addr = dc_exp, a0 = dc_exp, a1 = dc_exp + 1;
            bool busy = alive, b0 = false, b1 = busy;
            uint32_t mw = busy ? model[addr] : 0u;
            while (__any_sync(FULL, busy)) {
                if (busy) {
                    uint32_t split;
                    const uint32_t bit = g2_bit(br, s_rcp, mw, split);
                    const uint32_t naddr = bit ? a1 : a0;
                    const bool nbusy = bit ? b1 : b0;
                    uint32_t mwn = nbusy ? model[naddr] : 0u;
                    const uint32_t neww = g2_model_word(mw, bit);
                    model[addr] = (uint16_t)neww;
                    if (naddr == addr) mwn = neww;
                    g2_update(br, split, bit);
                    ++nd;
                    const int isE = st == G2_EXP, isS = st == G2_SIGN, isR = st == G2_RES;
                    const int cont = isE & (int)bit & (int)(len < 10);
                    const int len1 = len + (isE & (int)bit);
                    const int toS = isE & (cont ^ 1) & (int)(len1 != 0);
                    const int ris = len - 2;
                    const int evS = isS & (int)(ris < 0), toR = isS & (int)(ris >= 0);
                    const int evR = isR & (int)(ri == 0);
                    const int nval = isS ? (1 << ((len - 1) & 31)) : (isR ? (val | ((int)bit << (ri & 31))) : val);
                    const bool nneg = isS ? !bit : neg;
                    if (evS | evR) dcv = nneg ? -nval : nval;
                    st = toS ? G2_SIGN : toR ? G2_RES : st;
                    len = len1;
                    ri = isS ? ris : ri - isR;
                    val = nval; neg = nneg; addr = naddr; busy = nbusy; mw = mwn;
                    if (busy) {
                        const bool inE = st == G2_EXP, inS = st == G2_SIGN;
                        const bool fin = inS ? len < 2 : ri == 0;
                        const uint32_t common = inS ? dc_res + (uint32_t)(len - 2) : addr - 1;
                        a1 = inE ? (len < 10 ? addr + 1 : dc_sign) : common;
                        a0 = inE ? dc_sign : common;
                        b1 = inE ? true : !fin;
                        b0 = inE ? len != 0 : !fin;
                    }
                }
            }
        }

        // ---- (7) neighbour summaries (block_context.hh:44-78), block store in aligned order, next block
        if (alive) {
            const int dc = (int)(int16_t)adv_unpredict((int)(int16_t)dcv, true, pred);            // decoder.cc:305-309
            if (sub == 0) rcur[0] = (int16_t)dc;
            const int16_t qdc = (int16_t)((uint32_t)q0 * (uint32_t)dc);
            for (int i = sub; i < 16; i += G) {
                if (i < 8) {   // right column -> the next block's left neighbour
                    const int16_t cur = gs.pix[i * 8 + 7], prev = gs.pix[i * 8 + 6];
                    const int16_t delta = (int16_t)(cur - prev);
                    gs.ledge[i] = (int16_t)(cur + half_rz16(delta) + 1024 + qdc);
                } else {       // bottom row -> the block below
                    const int j = i - 8;
                    const int16_t cur = gs.pix[56 + j], prev = gs.pix[48 + j];
                    const int16_t delta = (int16_t)(cur - prev);
                    redge[(size_t)x * 8 + j] = (int16_t)(cur + half_rz16(delta) + 1024 + qdc);
                }
            }
            if (sub == 0) rnz[x] = (uint8_t)nz;
            nz_left = nz;
        }
        ndec += nd;
        if (bad) {                        // report the inconsistent stream; the group takes the next segment at the top
            if (sub == 0) {
                sdp->status = ST_STREAM_INCONSISTENT;
                sdp->len = (uint32_t)(br.p - reinterpret_cast<const uint8_t*>(sdp->stream));
                sdp->ndecisions_lo = (uint32_t)ndec;
                sdp->ndecisions_hi = (uint32_t)(ndec >> 32);
            }
        }
        __syncwarp();
        if (alive) {
            uint32_t* dst = reinterpret_cast<uint32_t*>(rowp + (size_t)x * 64) + sub * (CPL / 2);
#pragma unroll
            for (int k = 0; k < CPL / 2; ++k) {
                const int a = sub * CPL + 2 * k;
                const uint32_t lo = (uint16_t)rcur[s_a2r[a]];
                const uint32_t hi = (uint16_t)rcur[s_a2r[a + 1]];
                dst[k] = lo | (hi << 16);
            }
            // a truncated image ends inside a row (component_size_in_blocks)
            if (x + 1 >= w || (uint32_t)((size_t)y * w + x + 1) >= (uint32_t)gp->trunc_bc[c]) {
                need_row = true;
            } else {                      // the 7x7 count tree of the next block is known now (phase (1b) with a left neighbour)
                const int nza = has_above ? (int)rnz[x + 1] : 0;
                cnt_addr = m_nz7(ci, s_nzbin[has_above ? (nza + nz + 2) / 4 : (nz + 1) / 2], 0, 0);
                nzt = g2_nz_top(model + cnt_addr);
                cnt_ready = true;
                ++x; pc ^= 1; pa ^= 1;
            }
        }
        __syncwarp();
    }
}

}  // namespace lepb200
