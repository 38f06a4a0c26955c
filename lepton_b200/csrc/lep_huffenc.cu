// lep_huffenc.cu -- sm_90a baseline Huffman ENCODER for the decode direction (SURVEY.md section 8(f) row 2):
// coefficient planes resident in HBM (just produced by the arithmetic decoder) -> the entropy-coded bytes of the JPEG
// scan, byte-stuffed, with restart markers -- so that the D2H copy carries JPEG bytes instead of 128 B per block.
//
// Reference semantics: recode_row_range / recode_one_mcu_row / encode_block_seq / escape_0xff_huffman_and_write
// (src/lepton/recoder.cc:472-545, 316-410, 245-313, 144-185).  Like the reference, the unit of parallelism is the Lepton
// thread-segment: its ThreadHandoff gives the bits already pending in the first byte (overhang), the DC predictors and
// the number of file bytes it covers, so segments are independent.  ONE WARP PER SEGMENT; inside a block the 32 lanes
// build the codewords of two zig-zag positions each, a prefix sum places them in a shared-memory bit buffer, complete
// bytes leave with their 0xFF stuffing through a second prefix sum.
#include "lep_common.cuh"
#include "lep_predict.cuh"

namespace lepb200 {

struct HEncTable { uint16_t code[256]; uint8_t len[256]; };      // DHT as code/length per symbol (build_huffcodes, jpgcoder.cc:5508-5540)

struct HEncImage {
    unsigned long long plane[3];
    unsigned long long out;          // device address of the scan bytes of this image
    int32_t ncmp, mcuh, mcuv, rsti, padbit;
    int32_t H[3], V[3], bch[3];
    int32_t dc_tab[3], ac_tab[3];
    uint32_t scan_len;               // bytes the whole scan must produce
};

struct HEncSeg {
    int32_t image;
    int32_t my0, my1;                // MCU rows [my0, my1)
    int16_t lastdc[3];
    uint8_t ov_bits, ov_byte;        // bits pending in the first byte (ThreadHandoff overhang)
    uint32_t out_off;                // first byte this segment writes, relative to the scan start
    uint32_t expect;                 // bytes it must write (0 = last segment: runs to scan_len)
    int32_t is_last;
    int32_t status;                  // out: 0 ok, 1 length mismatch
    uint32_t produced;               // out
    uint32_t adler;                  // out: Adler-32 (RFC 1950) of the bytes written, [out_off, out_off + produced)
};

constexpr int HENC_WARPS = 4;
constexpr int HENC_WORDS = 160;      // bit buffer per warp: flushed once it holds HENC_FLUSH_BITS; a block adds at most ~1800 bits
constexpr uint32_t HENC_FLUSH_BITS = 2560;
constexpr uint32_t ADLER_MOD = 65521;

static __constant__ uint8_t c_zz2al[64] = {
    49, 50, 57, 58, 0, 51, 52, 1, 2, 59, 60, 3, 4, 5, 53, 54, 6, 7, 8, 9, 61, 62, 10, 11,
    12, 13, 14, 55, 56, 15, 16, 17, 18, 19, 20, 63, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32,
    33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48};

// spread the 32 bits of x to the even bit positions of a 64-bit word
__device__ __forceinline__ unsigned long long spread_bits(uint32_t x) {
    unsigned long long v = x;
    v = (v | (v << 16)) & 0x0000ffff0000ffffull;
    v = (v | (v << 8)) & 0x00ff00ff00ff00ffull;
    v = (v | (v << 4)) & 0x0f0f0f0f0f0f0f0full;
    v = (v | (v << 2)) & 0x3333333333333333ull;
    v = (v | (v << 1)) & 0x5555555555555555ull;
    return v;
}

// OR `n` (<= 32) bits, MSB first, into the bit buffer at bit position `pos`
__device__ __forceinline__ void put_bits(uint32_t* buf, uint32_t pos, uint32_t value, int n) {
    if (n == 0) return;
    const unsigned long long v = (unsigned long long)value << (64 - n);      // left-aligned in 64 bits
    const uint32_t wi = pos >> 5, sh = pos & 31;
    const unsigned long long s = v >> sh;
    atomicOr(&buf[wi], (uint32_t)(s >> 32));
    if ((uint32_t)s) atomicOr(&buf[wi + 1], (uint32_t)s);
    if (sh && n + sh > 64) atomicOr(&buf[wi + 2], (uint32_t)(v << (64 - sh)));
}

__global__ void __launch_bounds__(HENC_WARPS * 32)
lep_huffencode_kernel(const HEncImage* __restrict__ images, HEncSeg* __restrict__ segs, int nseg, const HEncTable* __restrict__ tables) {
    __shared__ uint32_t s_buf[HENC_WARPS][HENC_WORDS];
    __shared__ int16_t s_blk[HENC_WARPS][64];
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    const int sidx = blockIdx.x * HENC_WARPS + wid;
    if (sidx >= nseg) return;
    HEncSeg& sg = segs[sidx];
    const HEncImage& im = images[sg.image];
    uint32_t* buf = s_buf[wid];
    int16_t* sblk = s_blk[wid];
    for (int i = lane; i < HENC_WORDS; i += 32) buf[i] = 0;
    const int za0 = c_zz2al[2 * lane], za1 = c_zz2al[2 * lane + 1];      // aligned indices of this lane's zig-zag positions 2l, 2l+1
    uint8_t* const out = reinterpret_cast<uint8_t*>(im.out);
    const uint32_t limit = im.scan_len;
    uint32_t opos = sg.out_off;                                           // next byte to write
    uint32_t nbit = sg.ov_bits;                                           // bits pending in the buffer
    if (lane == 0 && nbit) buf[0] = (uint32_t)(sg.ov_byte & (0xff00u >> nbit) & 0xffu) << 24;
    __syncwarp();
    int dc0 = sg.lastdc[0], dc1 = sg.lastdc[1], dc2 = sg.lastdc[2];
    const int ncmp = im.ncmp, mcuh = im.mcuh, rsti = im.rsti;
    int rstw = 0, cpos = 0;
    if (rsti > 0) { const int m0 = sg.my0 * mcuh; rstw = rsti - (m0 % rsti); cpos = m0 / rsti; }
    const int mcu_end = im.mcuv * mcuh;
    // Adler-32 of the written bytes, taken while they are in registers: each lane sums the bytes it writes (a) and each byte
    // times its position relative to out_off (p); stuffed zeros add nothing.  p is reduced once per flush (a lane adds at most
    // about 20 terms below 2^40 between reductions), a at the end (below 2^40 for any 32-bit segment length).
    unsigned long long ad_a = 0, ad_p = 0;

    // writes the complete bytes of the buffer (with 0xFF stuffing) and keeps the remaining bits
    auto flush = [&]() {
        const uint32_t nbytes = nbit >> 3;
        for (uint32_t base = 0; base < nbytes; base += 32) {
            const uint32_t i = base + lane;
            const bool act = i < nbytes;
            const uint32_t b = act ? (buf[i >> 2] >> (24 - 8 * (i & 3))) & 0xffu : 0u;
            const uint32_t ffm = __ballot_sync(FULL, act && b == 0xffu);
            const uint32_t dst = opos + (i - base) + __popc(ffm & ((1u << lane) - 1));
            if (act) {
                if (dst < limit) { out[dst] = (uint8_t)b; ad_a += b; ad_p += (unsigned long long)(dst - sg.out_off) * b; }
                if (b == 0xffu && dst + 1 < limit) out[dst + 1] = 0;
            }
            opos += min(32u, nbytes - base) + __popc(ffm);
        }
        ad_p %= ADLER_MOD;
        __syncwarp();
        // move the leftover bits to the front, clear the rest
        const uint32_t rem = nbit & 7;
        const uint32_t keep = rem ? ((buf[nbytes >> 2] >> (24 - 8 * (nbytes & 3))) & 0xffu & (0xff00u >> rem)) << 24 : 0u;
        __syncwarp();
        const uint32_t used = (nbit + 31) >> 5;
        for (uint32_t i = lane; i <= used && i < HENC_WORDS; i += 32) buf[i] = 0;
        __syncwarp();
        if (lane == 0) buf[0] = keep;
        nbit = rem;
        __syncwarp();
    };

    for (int my = sg.my0; my < sg.my1; ++my) {
        for (int mx = 0; mx < mcuh; ++mx) {
            for (int c = 0; c < ncmp; ++c) {
                const int H = im.H[c], V = im.V[c], W = im.bch[c];
                const HEncTable& dct = tables[im.dc_tab[c]];
                const HEncTable& act = tables[im.ac_tab[c]];
                const uint32_t* plane = reinterpret_cast<const uint32_t*>(im.plane[c]);
                for (int sy = 0; sy < V; ++sy)
                    for (int sx = 0; sx < H; ++sx) {
                        const size_t dpos = (size_t)(my * V + sy) * W + mx * H + sx;
                        const uint32_t wv = plane[dpos * 32 + lane];
                        sblk[2 * lane] = (int16_t)(wv & 0xffff); sblk[2 * lane + 1] = (int16_t)(wv >> 16);
                        __syncwarp();
                        int v0 = sblk[za0], v1 = sblk[za1];                       // zig-zag positions 2l and 2l+1
                        __syncwarp();
                        // DC difference replaces position 0
                        int dcbits = 0;
                        uint32_t dcval = 0;
                        if (lane == 0) {
                            const int last = c == 0 ? dc0 : (c == 1 ? dc1 : dc2);
                            const int16_t diff = (int16_t)(v0 - last);
                            const int s = bitlen((uint32_t)iabs(diff));
                            const uint32_t mag = (uint32_t)(diff > 0 ? diff : diff - 1) & ((1u << s) - 1u);
                            dcbits = dct.len[s] + s;
                            dcval = ((uint32_t)dct.code[s] << s) | mag;
                        }
                        const int dcv = __shfl_sync(FULL, v0, 0);
                        if (c == 0) dc0 = dcv; else if (c == 1) dc1 = dcv; else dc2 = dcv;
                        if (lane == 0) v0 = 0;
                        // zig-zag mask of the non-zero AC coefficients
                        const uint32_t m0 = __ballot_sync(FULL, v0 != 0), m1 = __ballot_sync(FULL, v1 != 0);
                        const unsigned long long nz = spread_bits(m0) | (spread_bits(m1) << 1);
                        // codeword(s) of this lane's two positions
                        int nb[2] = {0, 0}, zrl[2] = {0, 0};
                        uint32_t cw[2] = {0, 0};
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int v = h ? v1 : v0;
                            if (v != 0) {
                                const int z = 2 * lane + h;
                                const unsigned long long below = nz & ((1ull << z) - 1ull);
                                const int prev = below ? 63 - __clzll((long long)below) : 0;
                                const int run = z - prev - 1;
                                const int s = bitlen((uint32_t)iabs(v));
                                const uint32_t mag = (uint32_t)(v > 0 ? v : v - 1) & ((1u << s) - 1u);
                                const int sym = ((run & 15) << 4) | s;
                                zrl[h] = run >> 4;
                                nb[h] = act.len[sym] + s;
                                cw[h] = ((uint32_t)act.code[sym] << s) | mag;
                            }
                        }
                        const int zl = act.len[0xF0];
                        const uint32_t zc = act.code[0xF0];
                        const int lastnz = nz ? 63 - __clzll((long long)nz) : 0;
                        const int eobbits = (lane == 31 && lastnz != 63) ? act.len[0x00] : 0;
                        const int mine = dcbits + zrl[0] * zl + nb[0] + zrl[1] * zl + nb[1] + eobbits;
                        int total;
                        uint32_t pos = nbit + (uint32_t)warp_excl_scan(mine, lane, total);
                        if (dcbits) { put_bits(buf, pos, dcval, dcbits); pos += dcbits; }
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            for (int k = 0; k < zrl[h]; ++k) { put_bits(buf, pos, zc, zl); pos += zl; }
                            if (nb[h]) { put_bits(buf, pos, cw[h], nb[h]); pos += nb[h]; }
                        }
                        if (eobbits) put_bits(buf, pos, act.code[0x00], eobbits);
                        nbit += (uint32_t)total;
                        __syncwarp();
                        if (nbit >= HENC_FLUSH_BITS) flush();          // bytes leave in batches, not per block
                    }
            }
            // restart interval boundary (recoder.cc:381-397): pad, marker, predictors reset -- not after the last MCU
            const int mcu = my * mcuh + mx;
            if (rsti > 0 && mcu + 1 < mcu_end && --rstw == 0) {
                if (nbit & 7) {
                    // abitwriter::pad (bitops.hh:168-175): successive bits of the fill pattern, LSB first
                    const int need = 8 - (int)(nbit & 7);
                    uint32_t bits = 0;
                    for (int k = 0; k < need; ++k) bits = (bits << 1) | ((im.padbit >> k) & 1u);
                    if (lane == 0) put_bits(buf, nbit, bits, need);
                    nbit += need;
                    __syncwarp();
                }
                flush();                                                  // every pending byte goes out before the marker
                if (lane == 0) {
                    const uint32_t mk = 0xD0u + (cpos & 7), rel = opos - sg.out_off;
                    if (opos < limit) { out[opos] = 0xFF; ad_a += 0xFFu; ad_p += (unsigned long long)rel * 0xFFu; }
                    if (opos + 1 < limit) { out[opos + 1] = (uint8_t)mk; ad_a += mk; ad_p += (unsigned long long)(rel + 1) * mk; }
                }
                opos += 2;
                ++cpos;
                rstw = rsti;
                dc0 = dc1 = dc2 = 0;
            }
        }
    }
    if (sg.is_last && (nbit & 7)) {
        const int need = 8 - (int)(nbit & 7);
        uint32_t bits = 0;
        for (int k = 0; k < need; ++k) bits = (bits << 1) | ((im.padbit >> k) & 1u);
        if (lane == 0) put_bits(buf, nbit, bits, need);
        nbit += need;
        __syncwarp();
    }
    flush();                                                              // complete bytes; a non-last segment drops its last bits (the next one starts with them)
    ad_a = __reduce_add_sync(FULL, (unsigned)(ad_a % ADLER_MOD));           // 32 terms below 2^16 each
    ad_p = __reduce_add_sync(FULL, (unsigned)ad_p);
    if (lane == 0) {
        const uint32_t produced = opos - sg.out_off;
        sg.produced = produced;
        // bytes b_0 .. b_{n-1}: A = 1 + sum b_i, B = n + sum (n - i) b_i = n + n (A - 1) - sum i b_i  (mod 65521)
        const unsigned long long n = produced % ADLER_MOD, a = ad_a % ADLER_MOD, p = ad_p % ADLER_MOD;
        const uint32_t A = (uint32_t)((1 + a) % ADLER_MOD);
        const uint32_t B = (uint32_t)((n + n * a + ADLER_MOD - p) % ADLER_MOD);
        sg.adler = (B << 16) | A;
        const uint32_t want = sg.is_last ? limit - sg.out_off : sg.expect;
        sg.status = produced == want ? 0 : 1;
    }
}

}  // namespace lepb200
