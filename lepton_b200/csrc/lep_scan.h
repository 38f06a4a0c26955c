// lep_scan.h -- host JPEG pieces shared by the front end (lep_jpeg.cc) and the re-encoders (lep_recode.cc): the header
// segment reader for DHT / DRI / SOS, the scan order walkers, and the block masks of the coefficient loops.
#pragma once
#include <emmintrin.h>

#include <cstring>
#include <vector>

#include "lep_host.h"

namespace lephost {

// The tables below are shared by every file that includes this header.  Hidden visibility lets the library reach them
// PC-relative, as it reaches file-local tables, instead of through the GOT inside the decode and encode loops.
#pragma GCC visibility push(hidden)

// zig-zag position -> AlignedBlock index (src/vp8/util/aligned_block.hh:56-65)
inline constexpr uint8_t k_zigzag_to_aligned[64] = {
    49, 50, 57, 58, 0, 51, 52, 1, 2, 59, 60, 3, 4, 5, 53, 54, 6, 7, 8, 9, 61, 62, 10, 11,
    12, 13, 14, 55, 56, 15, 16, 17, 18, 19, 20, 63, 21, 22, 23, 24, 25, 26, 27, 28, 29, 30, 31, 32,
    33, 34, 35, 36, 37, 38, 39, 40, 41, 42, 43, 44, 45, 46, 47, 48};

inline int be16(const uint8_t* p) { return (p[0] << 8) | p[1]; }

// Bit permutation from AlignedBlock order to zig-zag order, one byte of the mask at a time (built by the compiler).
struct ZzPermTable {
    uint64_t t[8][256] = {};
    constexpr ZzPermTable() {
        int al2zz[64] = {};
        for (int z = 0; z < 64; ++z) al2zz[k_zigzag_to_aligned[z]] = z;
        for (int byte = 0; byte < 8; ++byte)
            for (int v = 0; v < 256; ++v) {
                uint64_t m = 0;
                for (int bb = 0; bb < 8; ++bb) if (v & (1 << bb)) m |= 1ull << al2zz[byte * 8 + bb];
                t[byte][v] = m;
            }
    }
};
inline constexpr ZzPermTable g_zzperm{};

#pragma GCC visibility pop

inline uint64_t aligned_to_zigzag(uint64_t nz) {
    uint64_t m = 0;
    for (int byte = 0; byte < 8; ++byte) m |= g_zzperm.t[byte][(nz >> (8 * byte)) & 255];
    return m;
}

// zig-zag-ordered bit mask of the non-zero coefficients of an AlignedBlock (SSE2 compare + fixed bit permutation)
inline uint64_t nonzero_mask_zigzag(const int16_t* blk) {
    const __m128i zero = _mm_setzero_si128();
    uint64_t zmask = 0;                                   // bit a: coefficient a (aligned order) IS zero
    for (int i = 0; i < 4; ++i) {
        const __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i*>(blk + 16 * i));
        const __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i*>(blk + 16 * i + 8));
        zmask |= (uint64_t)(uint32_t)_mm_movemask_epi8(_mm_packs_epi16(_mm_cmpeq_epi16(a, zero), _mm_cmpeq_epi16(b, zero))) << (16 * i);
    }
    return aligned_to_zigzag(~zmask);
}

// bit z set when |coefficient at zig-zag position z| >= thr (thr in 1..32768): the positions a progressive
// scan at successive-approximation bit `sal` sees as non-zero (thr = 1 << sal) or as already significant
// (thr = 2 << sal)
inline uint64_t magnitude_mask_zigzag(const int16_t* blk, int thr) {
    const __m128i zero = _mm_setzero_si128();
    const __m128i t1 = _mm_set1_epi16((short)(thr - 1));
    uint64_t zmask = 0;                                   // bit a: |coefficient a| < thr
    for (int i = 0; i < 4; ++i) {
        __m128i a = _mm_loadu_si128(reinterpret_cast<const __m128i*>(blk + 16 * i));
        __m128i b = _mm_loadu_si128(reinterpret_cast<const __m128i*>(blk + 16 * i + 8));
        a = _mm_max_epi16(a, _mm_sub_epi16(zero, a));     // |x| as u16 (-32768 stays 0x8000 = 32768)
        b = _mm_max_epi16(b, _mm_sub_epi16(zero, b));
        const __m128i eq = _mm_packs_epi16(_mm_cmpeq_epi16(_mm_subs_epu16(a, t1), zero),
                                           _mm_cmpeq_epi16(_mm_subs_epu16(b, t1), zero));
        zmask |= (uint64_t)(uint32_t)_mm_movemask_epi8(eq) << (16 * i);
    }
    return aligned_to_zigzag(~zmask);
}

// Parameters of one scan: its components (frame indices, scan order), spectral band and successive approximation bits.
struct ScanInfo {
    int ncomp = 0;
    int cmp[4] = {0, 0, 0, 0};
    int from = 0, to = 0, sah = 0, sal = 0;
};

// Huffman tables and restart interval as the header segments read so far leave them, and the table selectors of each
// frame component as the last SOS naming it set them.
struct ScanTables {
    HuffTable dc[4], ac[4];
    int rsti = 0;
    int td[4] = {0, 0, 0, 0}, ta[4] = {0, 0, 0, 0};
    int ndef = 0;                    // DHT and DRI segments read
};

enum class Seg { sos, end, error };

// The marker segment at `pos` of a header blob (FF, type, two length bytes, payload): its type and its length with the
// marker counted.  False when fewer than four bytes are left.  The length may run past the end of an untrusted blob.
inline bool segment_at(const std::vector<uint8_t>& h, size_t pos, uint8_t& type, size_t& len) {
    if (pos + 4 > h.size()) return false;
    type = h[pos + 1];
    len = 2 + be16(&h[pos + 2]);
    return true;
}

// parse_jfif_jpg (jpgcoder.cc:4545-4680) for DHT, DRI and SOS: reads j.hdr from `pos` up to and including the next SOS.
// Returns Seg::sos with `pos` behind the SOS and `sc` filled, Seg::end with `pos` at the < 4 bytes left when there is no
// further SOS, or Seg::error with `err` set.  Nothing outside a segment is read: a DRI shorter than its two bytes reads
// zero for the missing ones, like the reference; everything else short is refused.
inline Seg read_to_sos(const Jpeg& j, size_t& pos, ScanTables& t, ScanInfo& sc, const char*& err) {
    const std::vector<uint8_t>& h = j.hdr;
    uint8_t type;
    size_t len;
    while (segment_at(h, pos, type, len)) {
        if (pos + len > h.size()) { err = "truncated header segment"; return Seg::error; }      // the header of a .lep is untrusted input
        const uint8_t* seg = &h[pos];
        pos += len;
        if (type == 0xC4) {
            ++t.ndef;
            // a class or id out of range ends the table list short of the segment's end: "size mismatch" (jpgcoder.cc:4558-4590)
            for (size_t p = 4; p < len;) {
                const int tc = seg[p] >> 4, th = seg[p] & 15;
                if (tc >= 2 || th >= 4 || p + 17 > len) { err = "size mismatch in dht marker"; return Seg::error; }
                ++p;
                HuffTable& ht = tc ? t.ac[th] : t.dc[th];
                ht = HuffTable();
                int total = 0;
                for (int i = 0; i < 16; ++i) { ht.bits[i + 1] = seg[p + i]; total += seg[p + i]; }
                if (total > 256 || p + 16 + total > len) { err = "size mismatch in dht marker"; return Seg::error; }
                memcpy(ht.vals, seg + p + 16, total);
                if (!ht.build()) { err = "bad huffman table"; return Seg::error; }
                ht.set = true;
                p += 16 + total;
            }
        } else if (type == 0xDD) {
            ++t.ndef;
            t.rsti = ((len > 4 ? seg[4] : 0) << 8) | (len > 5 ? seg[5] : 0);          // jpgcoder.cc:4621-4623
        } else if (type == 0xDA) {
            sc = ScanInfo();
            sc.ncomp = len > 4 ? seg[4] : 0;
            if (sc.ncomp < 1 || sc.ncomp > j.ncmp || len < (size_t)(8 + 2 * sc.ncomp)) { err = "bad SOS"; return Seg::error; }
            for (int i = 0; i < sc.ncomp; ++i) {
                int c = 0;
                while (c < j.ncmp && j.cmp[c].jid != seg[5 + 2 * i]) ++c;
                if (c == j.ncmp) { err = "component id mismatch in start-of-scan"; return Seg::error; }
                sc.cmp[i] = c;
                t.td[c] = seg[6 + 2 * i] >> 4;
                t.ta[c] = seg[6 + 2 * i] & 15;
                if (t.td[c] >= 4 || t.ta[c] >= 4) { err = "huffman table number mismatch"; return Seg::error; }
            }
            const uint8_t* s = seg + 5 + 2 * sc.ncomp;
            sc.from = s[0]; sc.to = s[1]; sc.sah = s[2] >> 4; sc.sal = s[2] & 15;
            if (sc.from > sc.to || sc.to > 63) { err = "spectral selection parameter out of range"; return Seg::error; }
            if (sc.sah >= 12 || sc.sal >= 12) { err = "successive approximation parameter out of range"; return Seg::error; }   // :4664-4668
            return Seg::sos;
        }
    }
    return Seg::end;
}

// rebuild_header_jpg (jpgcoder.cc:4848-4888), -d: the segments the coefficients are coded with -- DQT, DHT, DRI, SOF0-2
// and SOS -- in file order; everything else (APPn, COM, ...) is dropped.
inline std::vector<uint8_t> coding_segments(const std::vector<uint8_t>& h) {
    std::vector<uint8_t> out;
    out.reserve(h.size());
    uint8_t type;
    size_t len;
    for (size_t pos = 0; segment_at(h, pos, type, len) && pos + len <= h.size(); pos += len)
        if (type == 0xDA || type == 0xC4 || type == 0xDB || type == 0xC0 || type == 0xC1 || type == 0xC2 || type == 0xDD)
            out.insert(out.end(), h.begin() + pos, h.begin() + pos + len);
    return out;
}

// Every table the scan codes with is defined (jpgcoder.cc:2858-2868).
inline bool scan_tables_present(const Jpeg& j, const ScanTables& t, const ScanInfo& sc) {
    const bool need_dc = j.jpegtype == 1 || ((sc.ncomp > 1 || sc.to == 0) && sc.sah == 0);
    const bool need_ac = j.jpegtype == 1 || (sc.ncomp == 1 && sc.to > 0);
    for (int i = 0; i < sc.ncomp; ++i) {
        const int c = sc.cmp[i];
        if ((need_dc && !t.dc[t.td[c]].set) || (need_ac && !t.ac[t.ta[c]].set)) return false;
    }
    return true;
}

struct ScanPos {               // position bookkeeping shared by the scan walkers
    int cmp = 0, csc = 0, mcu = 0, sub = 0, dpos = 0, rstw = 0;
};

// next_mcupos (recoder.cc:190-243): interleaved order.  Returns 0 go on, 1 restart interval done, 2 scan done.
inline int next_mcupos(const Jpeg& j, const ScanInfo& sc, int rsti, ScanPos& p) {
    int sta = 0;
    if (++p.sub >= j.cmp[p.cmp].mbs) {
        p.sub = 0;
        if (++p.csc >= sc.ncomp) {
            p.csc = 0;
            p.cmp = sc.cmp[0];
            ++p.mcu;
            if (p.mcu >= j.mcuc) sta = 2;
            else if (rsti > 0 && --p.rstw == 0) sta = 1;
        } else {
            p.cmp = sc.cmp[p.csc];
        }
    }
    const Component& k = j.cmp[p.cmp];
    if (k.V > 1) {
        const int my = p.mcu / j.mcuh, mx = p.mcu - my * j.mcuh, sy = p.sub / k.H, sx = p.sub - sy * k.H;
        p.dpos = (my * k.V + sy) * k.bch + mx * k.H + sx;
    } else if (k.H > 1) {
        p.dpos = p.mcu * k.mbs + p.sub;
    } else {
        p.dpos = p.mcu;
    }
    return sta;
}

// next_mcuposn (jpgcoder.cc:5432-5456): single-component scan order over the non-padded blocks
inline int next_mcuposn(const Jpeg& j, int rsti, ScanPos& p) {
    const Component& k = j.cmp[p.cmp];
    p.dpos++;
    if (k.bch != k.nch && p.dpos % k.bch == k.nch) p.dpos += k.bch - k.nch;
    if (k.bcv != k.ncv && p.dpos / k.bch == k.ncv) p.dpos = k.bc;
    if (p.dpos >= k.bc) return 2;
    if (rsti > 0 && --p.rstw == 0) return 1;
    return 0;
}

}  // namespace lephost
