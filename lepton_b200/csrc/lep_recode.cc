// lep_recode.cc -- decode-side host halves: .lep container reader (read_ujpg, jpgcoder.cc:4117-4362; fixed header
// :2140-2176; MuxReader, src/io/MuxReader.hh:230-283; ThreadHandoff::deserialize, thread_handoff.cc:4-39) and the
// baseline JPEG re-creation from coefficient planes (recode_baseline_jpeg, src/lepton/recoder.cc:694-889;
// recode_one_mcu_row :316-410; encode_block_seq :245-313; 0xff stuffing :144-185).
//
// The reference re-encodes every thread-segment independently from its handoff (overhang bits + last DCs) and
// concatenates; encoding the scan front to back from the complete planes yields the same bytes, so that is what
// is done here (one host thread per file; files are processed in parallel by the caller).
#include <zlib.h>
#include <dlfcn.h>

#include <algorithm>
#include <cstring>
#include <mutex>

#include "lep_scan.h"

namespace lephost {

namespace {
inline uint32_t rd32(const uint8_t* p) { return p[0] | (p[1] << 8) | (p[2] << 16) | ((uint32_t)p[3] << 24); }
bool lfail(LepFile& lf, int st, const char* msg) { lf.status = st; lf.error = msg; return false; }

// Header blobs of container versions 2, 3 and 4 are brotli streams (write_ujpg, jpgcoder.cc:4032-4041; read_ujpg :4168-4175;
// the reference vendors the brotli sources).  Brotli needs the 122 KB static dictionary of RFC 7932, which is third-party
// DATA, so no decoder is written here: the system's libbrotlidec (the same kind of dependency as -lz for version 1) is
// loaded at run time through its stable streaming C API.  Without the library such files are refused (status 200) as before.
struct BrotliApi {
    void* (*create)(void*, void*, void*) = nullptr;
    int (*stream)(void*, size_t*, const uint8_t**, size_t*, uint8_t**, size_t*) = nullptr;
    void (*destroy)(void*) = nullptr;
    bool ok = false;
};
const BrotliApi& brotli_api() {
    static BrotliApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = nullptr;
        for (const char* name : {"libbrotlidec.so.1", "libbrotlidec.so"}) { h = dlopen(name, RTLD_NOW | RTLD_LOCAL); if (h) break; }
        if (!h) return;
        api.create = reinterpret_cast<void* (*)(void*, void*, void*)>(dlsym(h, "BrotliDecoderCreateInstance"));
        api.stream = reinterpret_cast<int (*)(void*, size_t*, const uint8_t**, size_t*, uint8_t**, size_t*)>(dlsym(h, "BrotliDecoderDecompressStream"));
        api.destroy = reinterpret_cast<void (*)(void*)>(dlsym(h, "BrotliDecoderDestroyInstance"));
        api.ok = api.create && api.stream && api.destroy;
    });
    return api;
}
// 0 ok, 1 no library, 2 corrupt stream, 3 larger than `cap`
int brotli_decompress(const uint8_t* in, size_t n, std::vector<uint8_t>& out, size_t cap) {
    const BrotliApi& b = brotli_api();
    if (!b.ok) return 1;
    void* st = b.create(nullptr, nullptr, nullptr);
    if (!st) return 1;
    out.resize(std::max<size_t>(4096, n * 6));
    size_t avail_in = n, have = 0;
    const uint8_t* next_in = in;
    int rc = 2;
    for (;;) {
        size_t avail_out = out.size() - have;
        uint8_t* next_out = out.data() + have;
        const int r = b.stream(st, &avail_in, &next_in, &avail_out, &next_out, nullptr);
        have = out.size() - avail_out;
        if (r == 1) { rc = 0; break; }                     // BROTLI_DECODER_RESULT_SUCCESS
        if (r != 3) { rc = 2; break; }                     // error, or more input wanted than the blob has
        if (out.size() >= cap) { rc = 3; break; }          // BROTLI_DECODER_RESULT_NEEDS_MORE_OUTPUT
        out.resize(std::min(cap, out.size() * 2));
    }
    b.destroy(st);
    out.resize(rc == 0 ? have : 0);
    return rc;
}

}  // namespace

bool brotli_available() { return brotli_api().ok; }

namespace {
bool read_container(const uint8_t* d, size_t n, LepFile& lf, bool lazy, std::vector<uint8_t>* carry) {
    // CF 84 (tau): the usual container; CE B6 (zeta, zlepton_header, jpgcoder.cc:552): the same container whose JPEG is handed
    // out as a zlib stream (check_file, jpgcoder.cc:2200-2220)
    const bool zeta = n >= 2 && d[0] == 0xCE && d[1] == 0xB6;
    if (n < 28 + 3 + 4 || !((d[0] == 0xCF && d[1] == 0x84) || zeta)) return lfail(lf, VERSION_UNSUPPORTED, "not a .lep file");
    lf.zlib0 = zeta;
    lf.version = d[2]; lf.flag = d[3]; lf.nseg = d[4];
    // version 1: zlib header blob; 2 and 4: brotli header blob (and an EOF marker behind the mux packets); 3: the same as 2 with
    // the rANS coder instead of the bool coder in every segment stream (makeDecoder(..., ujgversion == 3), jpgcoder.cc:1727)
    if (lf.version < 1 || lf.version > 4) return lfail(lf, NOT_HANDLED, "container version not handled");
    lf.jpeg_size = rd32(d + 20);
    const uint32_t zlen = rd32(d + 24);
    if ((size_t)28 + zlen + 3 + 4 > n) return lfail(lf, SHORT_READ, "truncated .lep");
    // inflate the header blob
    std::vector<uint8_t> blob;
    if (carry && !carry->empty()) {
        // -lepcat: the first member's blob holds the headers of the members behind it, and theirs are empty (read_ujpg :4187-4189)
        if (zlen != 0) return lfail(lf, ASSERTION_FAILURE, "Special concatenation requires 0 size header");
        blob.swap(*carry);
    } else if (lf.version != 1) {
        const int rc = brotli_decompress(d + 28, zlen, blob, size_t(256) << 20);
        if (rc == 1) return lfail(lf, NOT_HANDLED, "brotli header blob (container version 2 / 3 / 4) and no libbrotlidec on this system");
        if (rc == 3) return lfail(lf, 38 /*TOO_MUCH_MEMORY_NEEDED*/, "header blob too large");
        // version 3 whose blob is not brotli: refused as not handled, where the reference asserts (DESIGN section 6)
        if (rc && lf.version == 3) return lfail(lf, NOT_HANDLED, "container version 3 (rANS coder) whose header blob is not brotli coded");
        if (rc) return lfail(lf, ASSERTION_FAILURE, "Data not properly brotli coded");
    } else {
        z_stream zs;
        memset(&zs, 0, sizeof(zs));
        if (inflateInit(&zs) != Z_OK) return lfail(lf, ASSERTION_FAILURE, "inflateInit failed");
        zs.next_in = const_cast<uint8_t*>(d + 28); zs.avail_in = zlen;
        blob.resize(std::max<size_t>(4096, (size_t)zlen * 4));
        size_t have = 0;
        int ret;
        do {
            if (have == blob.size()) {
                // untrusted input: a few KB of zlib can expand to gigabytes.  The blob holds the JPEG header, garbage and
                // per-restart bookkeeping -- all bounded by the JPEG it describes (the reference bounds it through its
                // memory limit); 256 MB is far beyond any file the 4-byte size fields can describe sensibly
                if (blob.size() >= (size_t(256) << 20)) { inflateEnd(&zs); return lfail(lf, 38 /*TOO_MUCH_MEMORY_NEEDED, memory.hh:34*/, "header blob too large"); }
                blob.resize(blob.size() * 2);
            }
            zs.next_out = blob.data() + have; zs.avail_out = (uInt)(blob.size() - have);
            ret = inflate(&zs, Z_NO_FLUSH);
            have = blob.size() - zs.avail_out;
        } while (ret == Z_OK);
        inflateEnd(&zs);
        if (ret != Z_STREAM_END) return lfail(lf, ASSERTION_FAILURE, "Data not properly zlib coded");
        blob.resize(have);
    }
    if (carry) carry->clear();
    size_t p = 0;
    auto need = [&](size_t k) { return p + k <= blob.size(); };
    if (!need(7) || memcmp(&blob[p], "HDR", 3)) return lfail(lf, UNSUPPORTED_JPEG, "HDR marker not found");
    const uint32_t hdrs = rd32(&blob[p + 3]);
    p += 7;
    if (!need(hdrs)) return lfail(lf, SHORT_READ, "short HDR");
    Jpeg& j = lf.j;
    j.hdr.assign(blob.begin() + p, blob.begin() + p + hdrs);
    p += hdrs;
    if (!parse_frame(j)) { lf.status = j.status; lf.error = j.error; return false; }
    if (!need(4)) return lfail(lf, SHORT_READ, "short pad section");
    if (!memcmp(&blob[p], "P0D", 3)) {
        j.padbit = (int8_t)blob[p + 3];
    } else if (!memcmp(&blob[p], "PAD", 3)) {
        // legacy: one pad bit that stands for all of them (jpgcoder.cc:4228-4242)
        const int8_t pb = (int8_t)blob[p + 3];
        if (!(pb == 0 || pb == 1 || pb == -1)) return lfail(lf, STREAM_INCONSISTENT, "Legacy Padbit must be 0, 1 or -1");
        j.padbit = pb == 1 ? 0x7f : pb;
    } else {
        return lfail(lf, UNSUPPORTED_JPEG, "PAD marker not found");
    }
    p += 4;
    j.grb.clear();
    bool have_grb = false;
    while (need(3)) {
        const uint8_t* m = &blob[p];
        if (!memcmp(m, "CRS", 3)) {
            if (!need(7)) return lfail(lf, SHORT_READ, "short CRS");
            uint32_t k = rd32(m + 3);
            if (!need(7 + 4 * (size_t)k)) return lfail(lf, SHORT_READ, "short CRS");
            j.rst_cnt.resize(k);
            for (uint32_t i = 0; i < k; ++i) j.rst_cnt[i] = rd32(m + 7 + 4 * i);
            lf.rst_cnt_set = true;
            p += 7 + 4 * (size_t)k;
        } else if (m[0] == 'H' && m[1] == 'H') {
            const int k = m[2];
            if (!need(3 + 16 * (size_t)k)) return lfail(lf, VERSION_UNSUPPORTED, "short handoff table");
            for (int i = 0; i < k; ++i) {
                const uint8_t* r = m + 3 + 16 * i;
                Handoff h;
                h.luma_y_start = (uint16_t)(r[0] | (r[1] << 8));
                h.segment_size = rd32(r + 2);
                h.overhang_byte = r[6]; h.num_overhang_bits = r[7];
                for (int q = 0; q < 4; ++q) h.last_dc[q] = (int16_t)(r[8 + 2 * q] | (r[9 + 2 * q] << 8));
                lf.handoffs.push_back(h);
            }
            for (size_t i = 1; i < lf.handoffs.size(); ++i) lf.handoffs[i - 1].luma_y_end = lf.handoffs[i].luma_y_start;
            p += 3 + 16 * (size_t)k;
        } else if (!memcmp(m, "FRS", 3)) {
            if (!need(7)) return lfail(lf, SHORT_READ, "short FRS");
            uint32_t k = rd32(m + 3);
            if (!need(7 + (size_t)k)) return lfail(lf, SHORT_READ, "short FRS");
            j.rst_err.assign(m + 7, m + 7 + k);
            p += 7 + (size_t)k;
        } else if (!memcmp(m, "GRB", 3)) {
            if (!need(7)) return lfail(lf, SHORT_READ, "short GRB");
            uint32_t k = rd32(m + 3);
            if (!need(7 + (size_t)k)) return lfail(lf, SHORT_READ, "short GRB");
            j.grb.assign(m + 7, m + 7 + k);
            have_grb = true;
            p += 7 + (size_t)k;
        } else if (!memcmp(m, "EEE", 3)) {
            if (!need(31)) return lfail(lf, SHORT_READ, "short EEE");
            lf.has_eee = true;
            for (int i = 0; i < 7; ++i) lf.eee[i] = rd32(m + 3 + 4 * i);
            // UncompressedComponents::set_truncation_bounds (uncompressed_components.hh:166-188)
            j.early_eof = true;
            j.max_cmp = (int)lf.eee[0]; j.max_bpos = (int)lf.eee[1]; j.max_sah = (int)lf.eee[2];
            for (int c = 0; c < j.ncmp; ++c) {
                const Component& k = j.cmp[c];
                j.max_dpos[c] = (int)lf.eee[3 + c];
                const long tbc = (long)lf.eee[3 + c] + 1;
                if (tbc > k.bc) return lfail(lf, STREAM_INCONSISTENT, "truncation bound beyond the component");
                int vs = (int)std::min<long>(tbc / k.bch + (tbc % k.bch ? 1 : 0), k.bcv);
                const int ratio = k.bcv / j.mcuv;
                while (vs % ratio != 0 && vs + 1 <= k.bcv) ++vs;
                j.trunc_bcv[c] = vs;
                j.trunc_bc[c] = (int)tbc;
            }
            p += 31;
        } else if (!memcmp(m, "PGE", 3)) {
            // -embedding=N: the bytes in front of the embedded JPEG, written back in front of its SOI (read_ujpg :4292-4308)
            if (!need(7)) return lfail(lf, SHORT_READ, "short PGE");
            uint32_t k = rd32(m + 3);
            if (!need(7 + (size_t)k)) return lfail(lf, SHORT_READ, "short PGE");
            j.prefix.assign(m + 7, m + 7 + k);
            p += 7 + (size_t)k;
        } else if (carry && !memcmp(m, "CNT", 3)) {
            // -lepcat: this member's sections end here; the rest of the blob belongs to the members behind it (:4328-4330)
            carry->assign(m + 3, (const uint8_t*)blob.data() + blob.size());
            break;
        } else if (!memcmp(m, "PGR", 3) || !memcmp(m, "SIZ", 3)) {
            return lfail(lf, NOT_HANDLED, "-startbyte slice sections (PGR / SIZ) are not handled");
        } else {
            return lfail(lf, UNSUPPORTED_JPEG, "unknown data found in header blob");
        }
    }
    size_t q = 28 + (size_t)zlen;
    if (memcmp(d + q, "CMP", 3)) return lfail(lf, UNSUPPORTED_JPEG, "CMP marker missing");
    q += 3;
    const size_t end = n - 4;
    if (lf.flag == 'Y') {
        // Flag 'Y' is written by -permissive (generic_compress.cc:60-200) and by -startbyte slices.  Only the generic
        // container is taken: the fixed 1x1 grey header, zeroed handoffs, the whole file in PGE, an empty GRB and no coded
        // streams.  It restores to the PGE bytes, which the stored JPEG size bounds to exactly themselves.
        bool generic = j.hdr == generic_jpeg_header() && j.padbit == 0 && have_grb && j.grb.empty() && !lf.rst_cnt_set &&
                       j.rst_err.empty() && !lf.has_eee && j.prefix.size() == lf.jpeg_size && !j.prefix.empty() &&
                       !lf.handoffs.empty() && (int)lf.handoffs.size() == lf.nseg;
        for (const Handoff& h : lf.handoffs)
            generic = generic && !h.luma_y_start && !h.segment_size && !h.overhang_byte && !h.num_overhang_bits &&
                      !h.last_dc[0] && !h.last_dc[1] && !h.last_dc[2] && !h.last_dc[3];
        if (q + 3 <= end && d[q] == 0xFF && d[q + 1] == 0xFE && d[q + 2] == 0xFF) lf.member_end = q + 3;   // versions > 1: EOF marker
        else generic = generic && q == end;
        if (!generic) return lfail(lf, NOT_HANDLED, "'Y' container other than the generic one (-startbyte slices) not handled");
        lf.generic = true;
        lf.nseg = 0;
        lf.handoffs.clear();
        return true;
    }
    if (!have_grb) { j.grb = {0xFF, 0xD9}; }          // "if we don't have any garbage, assume FFD9 EOI" (jpgcoder.cc:4194)
    if (lf.handoffs.empty()) {
        // Legacy files (before the handoff table existed): the payload opens with the number of thread-segments and
        // the luma rows where they end (VP8ComponentDecoder::initialize_baseline_decoder, vp8_decoder.cc:337-369).
        // Their handoffs carry no Huffman state (ThreadHandoff::LEGACY_OVERHANG_BITS), so the scan can only be
        // re-created front to back -- which is what the host re-encoder does anyway.
        if (q + 1 > end) return lfail(lf, SHORT_READ, "legacy segment table missing");
        const int k = d[q];
        if (k == 0) return lfail(lf, THREADING_PARTIAL_MCU, "legacy segment count is zero");
        if (q + 1 + 2 * (size_t)(k - 1) > end) return lfail(lf, SHORT_READ, "short legacy segment table");
        const int luma_mul = j.cmp[0].bcv / j.mcuv;
        for (int i = 0; i < k; ++i) {
            Handoff h;
            h.num_overhang_bits = 0xff;
            h.luma_y_end = i + 1 < k ? (uint16_t)(d[q + 1 + 2 * i] | (d[q + 2 + 2 * i] << 8)) : (uint16_t)j.cmp[0].bcv;
            if (i + 1 < k && h.luma_y_end % luma_mul) return lfail(lf, THREADING_PARTIAL_MCU, "legacy split inside an MCU row");
            h.luma_y_start = i ? lf.handoffs[i - 1].luma_y_end : 0;
            lf.handoffs.push_back(h);
        }
        q += 1 + 2 * (size_t)(k - 1);
        lf.nseg = k;
        lf.legacy = true;
    }
    if ((int)lf.handoffs.size() != lf.nseg) return lfail(lf, VERSION_UNSUPPORTED, "handoff table inconsistent with the thread count");
    if (lf.nseg > 16) return lfail(lf, NOT_HANDLED, "more than 16 thread-segments");             // MAX_NUM_THREADS of this build
    // a corrupt handoff table must fail this file only, not the batch it travels in
    if (lf.handoffs[0].luma_y_start != 0) return lfail(lf, STREAM_INCONSISTENT, "first thread-segment does not start at row 0");
    for (int i = 0; i < lf.nseg; ++i) {
        if ((int)lf.handoffs[i].luma_y_start > j.cmp[0].bcv || (i + 1 < lf.nseg && lf.handoffs[i].luma_y_start > lf.handoffs[i + 1].luma_y_start))
            return lfail(lf, STREAM_INCONSISTENT, "thread-segment rows out of order or beyond the image");
    }
    // demux (src/io/MuxReader.hh:230-283); the last 4 bytes are the file-size trailer
    if (lazy) { lf.spans.assign(16, {}); lf.stream_len.assign(16, 0); }
    else lf.streams.assign(16, std::vector<uint8_t>());
    lf.member_end = 0;
    while (q + 3 <= end) {
        if (d[q] == 0xFF && d[q + 1] == 0xFE && d[q + 2] == 0xFF) { lf.member_end = q + 3; break; }   // MuxReader::getEofMarker (MuxReader.hh:131-139,240-243), written by versions > 1
        const uint8_t hd = d[q];
        const int sid = hd & 15, flags = (hd >> 4) & 3;
        size_t len, skip;
        if (flags == 0) { len = (size_t)d[q + 1] + 256 * (size_t)d[q + 2] + 1; skip = 3; }
        else { len = (size_t)1024 << (2 * flags); skip = 1; }
        if (q + skip + len > end) return lfail(lf, SHORT_READ, "mux packet runs past the end of the file");
        if (lazy) { lf.spans[sid].emplace_back(d + q + skip, (uint32_t)len); lf.stream_len[sid] += len; }
        else lf.streams[sid].insert(lf.streams[sid].end(), d + q + skip, d + q + skip + len);
        q += skip + len;
    }
    if (lazy) { lf.spans.resize(lf.nseg); lf.stream_len.resize(lf.nseg); }
    else lf.streams.resize(lf.nseg);
    return true;
}

}  // namespace

bool read_lep(const uint8_t* d, size_t n, LepFile& lf, bool lazy, std::vector<uint8_t>* carry) {
    if (read_container(d, n, lf, lazy, carry)) return true;
    // a 'Y' container that is not the generic one is a -startbyte slice, whatever else is wrong with it
    if (lf.flag == 'Y' && lf.status != NOT_HANDLED) { lf.status = NOT_HANDLED; lf.error = "'Y' container (-startbyte slice) not handled: " + lf.error; }
    return false;
}

void read_lep_members(const uint8_t* d, size_t n, std::vector<std::unique_ptr<LepFile>>& out, bool lazy) {
    out.clear();
    std::vector<uint8_t> carry;            // -lepcat: header sections of the members still to come
    bool baseline_only = false;            // g_allow_progressive turned off by a member's flag (read_fixed_ujpg_header :2162-2166)
    size_t o = 0;
    for (;;) {
        out.emplace_back(new LepFile());
        LepFile& lf = *out.back();
        if (!read_lep(d + o, n - o, lf, lazy, &carry)) return;
        // A progressive member behind a 'Z' one is handed to the reference's baseline re-encoder, which asserts on it
        // (recoder.cc:639, tests/golden/concat.json "baseline_then_progressive")
        if (lf.flag == 'X' && baseline_only) { lfail(lf, ASSERTION_FAILURE, "progressive member behind a baseline one"); return; }
        baseline_only |= lf.flag == 'Z' || (lf.flag & 1);
        // version 1 has no EOF marker: the reference's mux reader takes everything up to the end of the stream
        if (lf.member_end == 0) return;
        // the 4-byte size trailer (not checked), then the magic of the next member: fewer than 6 bytes, or other magic
        // bytes than the first member's, end the stream and the rest is ignored (process_file :1876-1896)
        const size_t next = o + lf.member_end + 4;
        if (next + 2 > n || d[next] != d[0] || d[next + 1] != d[1]) return;
        o = next;
    }
}

// ------------------------------------------------------------------------------------------------
// Huffman re-encoding of the (single, interleaved or single-component) baseline scan
// ------------------------------------------------------------------------------------------------
namespace {

inline int bitlen16(int v) { return v ? 32 - __builtin_clz((unsigned)v) : 0; }

// Bit writer of the baseline re-encoder (the hot loop of the .lep -> JPEG direction on the host): 64-bit accumulator,
// four bytes leave at a time unless one of them is 0xFF and needs its stuffed zero (recoder.cc:144-185).
struct FastWriter {
    std::vector<uint8_t>& out;
    uint8_t* p;
    uint8_t* lim;
    uint64_t acc = 0;
    int nbits = 0;
    explicit FastWriter(std::vector<uint8_t>& o, size_t expect) : out(o) {
        const size_t used = out.size();
        out.resize(used + expect + 4096);
        p = out.data() + used; lim = out.data() + out.size();
    }
    inline void room(size_t n) {
        if ((size_t)(lim - p) >= n) return;
        const size_t used = (size_t)(p - out.data());
        out.resize(out.size() * 2 + n + 4096);
        p = out.data() + used; lim = out.data() + out.size();
    }
    inline void raw(uint8_t b) { room(1); *p++ = b; }
    inline void raw_bytes(const uint8_t* src, size_t n) { room(n); memcpy(p, src, n); p += n; }
    inline void put(uint32_t v, int n) {          // n <= 32, v < 2^n
        if (n > 32) n = 32;                       // tables are validated by HuffTable::build(); never shift by >= 64
        acc = (acc << n) | v;
        nbits += n;
        if (nbits >= 32) {
            const uint32_t w = (uint32_t)(acc >> (nbits - 32));
            nbits -= 32;
            room(8);
            if (((w & 0x7f7f7f7fu) + 0x01010101u) & w & 0x80808080u) {          // some byte is 0xFF (exact test: b == 0xFF <=> (b & 0x7f) + 1 carries into a set top bit)
                for (int sh = 24; sh >= 0; sh -= 8) {
                    const uint8_t b = (uint8_t)(w >> sh);
                    *p++ = b;
                    if (b == 0xFF) *p++ = 0x00;
                }
            } else {
                p[0] = (uint8_t)(w >> 24); p[1] = (uint8_t)(w >> 16); p[2] = (uint8_t)(w >> 8); p[3] = (uint8_t)w;
                p += 4;
            }
        }
    }
    inline void flush_bytes() {
        room(16 + (size_t)(nbits / 8) * 2);
        while (nbits >= 8) {
            const uint8_t b = (uint8_t)(acc >> (nbits - 8));
            *p++ = b;
            if (b == 0xFF) *p++ = 0x00;
            nbits -= 8;
        }
    }
    // abitwriter::pad (bitops.hh:168-175): successive bits of `fill`, LSB first
    inline void pad(uint8_t fill) {
        int offset = 1;
        while (nbits & 7) { put((fill & offset) ? 1 : 0, 1); offset <<= 1; }
        flush_bytes();
    }
    inline void finish() { out.resize((size_t)(p - out.data())); }
};

// encode_block_seq (recoder.cc:245-313): the DC difference, then the run/size codes of the non-zero AC coefficients in
// zig-zag order.  Each code goes out with its magnitude bits in one put: at most 16 + 16 bits for any int16 coefficient.
inline void encode_block_seq(FastWriter& bw, const int16_t* blk, const HuffTable& dct, const HuffTable& act, int& lastdc) {
    const int16_t dc = blk[k_zigzag_to_aligned[0]];
    const int16_t diff = (int16_t)(dc - (int16_t)lastdc);
    lastdc = dc;
    int s = bitlen16(diff > 0 ? diff : -diff);
    int nb = diff > 0 ? diff : (diff - 1) + (1 << s);
    bw.put(((uint32_t)dct.ecode[s] << s) | (uint32_t)nb, dct.elen[s] + s);
    uint64_t m = nonzero_mask_zigzag(blk) >> 1;           // bit k: zig-zag position k + 1
    int prev = 0;
    while (m) {
        const int z = __builtin_ctzll(m) + 1;
        m &= m - 1;
        int run = z - prev - 1;
        prev = z;
        while (run >= 16) { bw.put(act.ecode[0xF0], act.elen[0xF0]); run -= 16; }
        const int v = blk[k_zigzag_to_aligned[z]];
        s = bitlen16(v > 0 ? v : -v);
        nb = v > 0 ? v : (v - 1) + (1 << s);
        const int hc = (run << 4) + s;
        bw.put(((uint32_t)act.ecode[hc] << s) | (uint32_t)nb, act.elen[hc] + s);
    }
    if (prev != 63) bw.put(act.ecode[0x00], act.elen[0x00]);
}

}  // namespace

bool recode_scans(const LepFile& lf, const int16_t* const planes[4], std::vector<uint8_t>& out, std::string& err);

namespace {
// A re-created JPEG of `n` bytes (counted with its prefix) against the size the container promises: the same, or shorter
// when the header holds nothing but the coding segments, as -d leaves it -- the container keeps the size of the file
// with its metadata, and the reference restores the file without it.
bool size_checks(const LepFile& lf, size_t n, std::string& err) {
    if (n == lf.jpeg_size || (n < lf.jpeg_size && coding_segments(lf.j.hdr).size() == lf.j.hdr.size())) return true;
    err = "re-created JPEG has the wrong size";
    return false;
}
}  // namespace

bool gpu_recode_setup(const LepFile& lf, GpuRecodeSetup& out) {
    const Jpeg& j = lf.j;
    if (lf.flag != 'Z' || lf.has_eee || !gpu_scan_setup(j, out, &out.hpos)) return false;
    for (int c = 0; c < j.ncmp; ++c) if (j.cmp[c].H < 1 || j.cmp[c].H > 2 || j.cmp[c].V < 1 || j.cmp[c].V > 2) return false;
    if (j.ncmp == 1 && (j.cmp[0].H != 1 || j.cmp[0].V != 1 || j.cmp[0].bch != j.cmp[0].nch || j.cmp[0].bcv != j.cmp[0].ncv)) return false;   // single-component scans walk nch x ncv blocks in raster order
    // every restart marker of the scan must be wanted (truncated originals limit them, recoder.cc:381-397)
    const unsigned nrst = out.rsti ? (unsigned)(j.mcuc - 1) / (unsigned)out.rsti : 0u;
    if (lf.rst_cnt_set && !j.rst_cnt.empty() && j.rst_cnt[0] < nrst) return false;
    const size_t trailing = j.rst_err.empty() ? 0 : 2 * (size_t)j.rst_err[0];
    const size_t fixed = j.prefix.size() + 2 + j.hdr.size() + j.grb.size() + trailing;
    if ((size_t)lf.jpeg_size <= fixed) return false;
    out.scan_bytes = (uint32_t)(lf.jpeg_size - fixed);
    return true;
}

namespace {
constexpr size_t ZLIB0_BLOCK = 65535;

// Writes the zlib0 stream of a payload of known length `n` that arrives in pieces: block headers go in where the payload
// crosses a block boundary, so every payload byte is copied exactly once.
struct Zlib0Writer {
    uint8_t* q = nullptr;
    size_t n = 0, pos = 0;            // payload length, payload bytes written so far
    bool sum = false;                 // take the Adler-32 of the pieces here
    uLong adler = 1;
    Zlib0Writer(std::vector<uint8_t>& out, size_t len, bool take_adler) : n(len), sum(take_adler) {
        out.resize(zlib0_size(len));
        q = out.data();
        *q++ = 0x78; *q++ = 0x01;     // CMF: deflate, 32 K window; FLG: no dictionary, fastest (check bits: 0x7801 % 31 == 0)
        if (n == 0) { *q++ = 1; *q++ = 0; *q++ = 0; *q++ = 0xFF; *q++ = 0xFF; }     // nothing to store: one empty final block
    }
    void put(const uint8_t* p, size_t len) {
        if (sum) adler = adler32(adler, p, (uInt)len);
        while (len) {
            if (pos % ZLIB0_BLOCK == 0) {
                const size_t b = std::min(ZLIB0_BLOCK, n - pos);
                q[0] = pos + b == n ? 1 : 0;
                q[1] = (uint8_t)b; q[2] = (uint8_t)(b >> 8); q[3] = (uint8_t)~b; q[4] = (uint8_t)(~b >> 8);
                q += 5;
            }
            const size_t k = std::min(len, ZLIB0_BLOCK - pos % ZLIB0_BLOCK);
            memcpy(q, p, k);
            q += k; p += k; pos += k; len -= k;
        }
    }
    void finish(uint32_t a) { q[0] = (uint8_t)(a >> 24); q[1] = (uint8_t)(a >> 16); q[2] = (uint8_t)(a >> 8); q[3] = (uint8_t)a; }
};
}  // namespace

size_t zlib0_size(size_t n) { return 2 + n + 5 * std::max<size_t>(1, (n + ZLIB0_BLOCK - 1) / ZLIB0_BLOCK) + 4; }

void zlib0_frame(const uint8_t* data, size_t n, std::vector<uint8_t>& out) {
    Zlib0Writer w(out, n, true);
    w.put(data, n);
    w.finish((uint32_t)w.adler);
}

void zlib0_join(const std::vector<std::pair<const uint8_t*, size_t>>& parts, const uint32_t* adlers, std::vector<uint8_t>& out) {
    size_t total = 0;
    for (const auto& pc : parts) total += pc.second;
    Zlib0Writer w(out, total, false);
    uLong a = 1;
    for (size_t k = 0; k < parts.size(); ++k) {
        w.put(parts[k].first, parts[k].second);
        a = adler32_combine(a, adlers[k], (z_off_t)parts[k].second);
    }
    w.finish((uint32_t)a);
}

bool assemble_baseline(const LepFile& lf, const GpuRecodeSetup& gs, const uint8_t* scan, std::vector<uint8_t>& out, std::string& err,
                       bool zlib0, uint32_t scan_adler, uint32_t* member_adler) {
    const Jpeg& j = lf.j;
    const std::vector<uint8_t>& h = j.hdr;
    static const uint8_t soi[2] = {0xFF, 0xD8};
    uint8_t rst[2 * 256];                                  // trailing restart markers (rst_err entries are bytes)
    size_t nrst = 0;
    if (!j.rst_err.empty()) {
        const unsigned cum = gs.rsti ? (unsigned)(j.mcuh * j.mcuv - 1) / gs.rsti : 0;
        for (unsigned i = 0; i < j.rst_err[0] && nrst + 2 <= sizeof(rst); ++i) { rst[nrst++] = 0xFF; rst[nrst++] = (uint8_t)(0xD0 + ((cum + i) & 7)); }
    }
    // the JPEG in pieces: [0, 3) in front of the scan (prefix of an embedded JPEG, SOI, header), [3] the scan, [4, 7) behind it
    const std::pair<const uint8_t*, size_t> pieces[7] = {
        {j.prefix.data(), j.prefix.size()}, {soi, 2}, {h.data(), gs.hpos}, {scan, gs.scan_bytes}, {rst, nrst},
        {h.data() + gs.hpos, h.size() - gs.hpos}, {j.grb.data(), j.grb.size()}};
    size_t total = 0;
    for (const auto& pc : pieces) total += pc.second;
    if (total != lf.jpeg_size) { err = "re-created JPEG has the wrong size"; out.clear(); return false; }
    // the device took the scan's sum; the host sums the few header and trailer bytes and combines the three
    auto adler = [&]() {
        uLong head = 1, tail = 1;
        size_t ntail = 0;
        for (int k = 0; k < 3; ++k) head = adler32(head, pieces[k].first, (uInt)pieces[k].second);
        for (int k = 4; k < 7; ++k) { tail = adler32(tail, pieces[k].first, (uInt)pieces[k].second); ntail += pieces[k].second; }
        return (uint32_t)adler32_combine(adler32_combine(head, scan_adler, (z_off_t)gs.scan_bytes), tail, (z_off_t)ntail);
    };
    if (!zlib0 || member_adler) {
        out.clear();
        out.reserve((size_t)lf.jpeg_size + 16);
        for (const auto& pc : pieces) out.insert(out.end(), pc.first, pc.first + pc.second);
        if (member_adler) *member_adler = adler();
        return true;
    }
    Zlib0Writer w(out, total, false);
    for (const auto& pc : pieces) w.put(pc.first, pc.second);
    w.finish(adler());
    return true;
}

bool recode_baseline(const LepFile& lf, const int16_t* const planes[4], std::vector<uint8_t>& out, std::string& err, bool zlib0,
                     uint32_t* member_adler) {
    if (zlib0 && member_adler) {
        if (!recode_baseline(lf, planes, out, err)) return false;
        *member_adler = (uint32_t)adler32(1, out.data(), (uInt)out.size());
        return true;
    }
    if (zlib0) {
        thread_local std::vector<uint8_t> jpeg;
        if (!recode_baseline(lf, planes, jpeg, err)) { out.clear(); return false; }
        zlib0_frame(jpeg.data(), jpeg.size(), out);
        return true;
    }
    const Jpeg& j = lf.j;
    if (lf.flag != 'Z' || j.jpegtype != 1) return recode_scans(lf, planes, out, err);     // multi-scan / progressive files
    const std::vector<uint8_t>& h = j.hdr;
    // handle_initial_segments (recoder.cc:412-461): everything up to and including the first SOS
    ScanTables t;
    ScanInfo sc;
    size_t hpos = 0;
    const char* msg = "overran headers";
    if (read_to_sos(j, hpos, t, sc, msg) != Seg::sos) { err = msg; return false; }
    if (!scan_tables_present(j, t, sc)) { err = "scan refers to a missing huffman table"; return false; }
    if (sc.ncomp != j.ncmp) { err = "non-interleaved multi-scan baseline not handled"; return false; }
    const int rsti = t.rsti;
    out.clear();
    out.reserve((size_t)lf.jpeg_size + 64);
    out.insert(out.end(), j.prefix.begin(), j.prefix.end());       // embedded JPEG: the prefix, then SOI and header (recoder.cc:449-456)
    out.push_back(0xFF); out.push_back(0xD8);
    out.insert(out.end(), h.begin(), h.begin() + hpos);

    FastWriter bw(out, (size_t)lf.jpeg_size);
    int lastdc[4] = {0, 0, 0, 0};
    const int mcuc = j.mcuc;
    unsigned rst_written = 0;
    const bool rst_limited = lf.rst_cnt_set && !j.rst_cnt.empty();
    ScanPos p;
    p.rstw = rsti;
    auto encode_block = [&](int c, int dpos) {
        encode_block_seq(bw, planes[c] + (size_t)dpos * 64, t.dc[t.td[c]], t.ac[t.ta[c]], lastdc[c]);
    };
    auto restart = [&]() {      // recoder.cc:381-397
        bw.pad((uint8_t)j.padbit);
        if (!rst_limited || rst_written < j.rst_cnt[0]) {
            bw.raw(0xFF);
            bw.raw((uint8_t)(0xD0 + (rst_written & 7)));
            rst_written++;
        }
        p.rstw = rsti;
        lastdc[0] = lastdc[1] = lastdc[2] = lastdc[3] = 0;
    };
    if (j.ncmp > 1) {
        // next_mcupos order, one MCU at a time
        for (int mcu = 0; mcu < mcuc; ++mcu) {
            const int my = mcu / j.mcuh, mx = mcu - my * j.mcuh;
            for (int ci = 0; ci < sc.ncomp; ++ci) {
                const int c = sc.cmp[ci];
                const Component& k = j.cmp[c];
                for (int sub = 0; sub < k.mbs; ++sub) {
                    const int sy = sub / k.H, sx = sub - sy * k.H;
                    encode_block(c, (my * k.V + sy) * k.bch + mx * k.H + sx);
                }
            }
            if (mcu + 1 < mcuc && rsti > 0 && --p.rstw == 0) restart();
        }
    } else {
        int sta = 0;
        while (sta != 2) {
            encode_block(0, p.dpos);
            sta = next_mcuposn(j, rsti, p);
            if (sta == 1) restart();
        }
    }
    bw.pad((uint8_t)j.padbit);
    // trailing bogus restart markers of the (only) scan (recoder.cc:839-848)
    if (!j.rst_err.empty()) {
        const unsigned cum = rsti ? (unsigned)(j.mcuh * j.mcuv - 1) / rsti : 0;
        for (unsigned i = 0; i < j.rst_err[0]; ++i) { bw.raw(0xFF); bw.raw((uint8_t)(0xD0 + ((cum + i) & 7))); }
    }
    bw.finish();
    out.insert(out.end(), h.begin() + hpos, h.end());      // header data after the first SOS, if any
    // everything before the garbage is bounded to (original size - garbage size): for truncated originals the scan is
    // cut exactly where the file ended (str_out->set_bound, recoder.cc:699-700, 880-886)
    if (lf.jpeg_size >= j.grb.size() && out.size() > lf.jpeg_size - j.grb.size()) out.resize(lf.jpeg_size - j.grb.size());
    out.insert(out.end(), j.grb.begin(), j.grb.end());
    return size_checks(lf, out.size(), err);
}


// ------------------------------------------------------------------------------------------------
// General (multi-scan) re-encoder for containers flagged 'X': progressive JPEGs and sequential files whose scans do
// not interleave every component.  Restates recode_jpeg (jpgcoder.cc:3309-3724) + the block routines
// (encode_dc_prg_fs :4993, encode_ac_prg_fs :5078, encode_dc_prg_sa :5137, encode_ac_prg_sa :5247, encode_eobrun :5346,
// encode_crbits :5379) and the marker/stuffing pass merge_jpeg_streaming (:2562-2740), fused into one front-to-back walk.
// ------------------------------------------------------------------------------------------------
namespace {

inline int fdiv2(int v, int p) { return v < 0 ? -((-v) >> p) : (v >> p); }

struct ProgWriter {
    FastWriter& bw;
    std::vector<uint32_t> crwords;        // stored correction bits (abytewriter "storw"), 32 to a word, oldest first
    uint32_t crcur = 0;
    int crn = 0;
    unsigned eobrun = 0;
    bool bad = false;                      // coefficients the scan's tables cannot express (inconsistent .lep)
    explicit ProgWriter(FastWriter& b) : bw(b) {}
    inline void push_crbit(uint32_t b) {
        crcur = (crcur << 1) | b;
        if (++crn == 32) { crwords.push_back(crcur); crcur = 0; crn = 0; }
    }
    void flush_crbits() {
        for (uint32_t w : crwords) bw.put(w, 32);
        crwords.clear();
        if (crn) { bw.put(crcur, crn); crcur = 0; crn = 0; }
    }
    void flush_eobrun(const HuffTable& t) {
        if (eobrun == 0) return;
        if (t.max_eobrun <= 0) { bad = true; eobrun = 0; return; }      // the table has no end-of-band code at all
        while (eobrun > (unsigned)t.max_eobrun) {
            bw.put(t.ecode[0xE0], t.elen[0xE0]);
            bw.put(32767 - (1 << 14), 14);
            eobrun -= (unsigned)t.max_eobrun;
        }
        int s = bitlen16((int)eobrun);
        if (s) --s;
        bw.put(t.ecode[s << 4], t.elen[s << 4]);
        bw.put(eobrun - (1u << s), s);
        eobrun = 0;
    }
};

}  // namespace

bool recode_scans(const LepFile& lf, const int16_t* const planes[4], std::vector<uint8_t>& out, std::string& err) {
    const Jpeg& j = lf.j;
    const std::vector<uint8_t>& h = j.hdr;
    ScanTables t;
    size_t hpos = 0;
    out.clear();
    out.reserve((size_t)lf.jpeg_size + 64);
    // no prefix: the reference's multi-scan restore (recode_jpeg / merge_jpeg_streaming, jpgcoder.cc:2562-2740, 3309) writes
    // SOI and header only, so an embedded progressive JPEG comes back without the bytes in front of it
    out.push_back(0xFF); out.push_back(0xD8);
    FastWriter bw(out, (size_t)lf.jpeg_size);
    ProgWriter pw(bw);
    bool rst_stuck = false;                // a refused marker is never retried (rpos stops advancing, :2640-2650)
    int scan = 0;
    while (true) {
        // ---- header segments up to and including the next SOS, copied as they are
        ScanInfo sc;
        const size_t seg_begin = hpos;
        const char* msg = nullptr;
        const Seg seg = read_to_sos(j, hpos, t, sc, msg);
        if (seg == Seg::error) { err = msg; return false; }
        bw.raw_bytes(h.data() + seg_begin, hpos - seg_begin);
        if (seg == Seg::end) break;
        ++scan;
        if (!scan_tables_present(j, t, sc)) { err = "huffman table missing in scan"; return false; }
        // ---- one scan
        const int rsti = t.rsti;
        unsigned cpos = 0, rst_this_scan = 0;
        auto rst_ok = [&]() {              // rst_cnt_ok (:2509-2517)
            if (rsti == 0 || rst_stuck) return false;
            if (!lf.rst_cnt_set) return true;
            return j.rst_cnt.size() > (size_t)scan - 1 && rst_this_scan < j.rst_cnt[scan - 1];
        };
        ScanPos p;
        p.cmp = sc.cmp[0];
        const bool inter = sc.ncomp > 1;
        auto coef = [&](int bpos) -> int { return planes[p.cmp][(size_t)p.dpos * 64 + k_zigzag_to_aligned[bpos]]; };
        auto next_pos = [&]() { return inter ? next_mcupos(j, sc, rsti, p) : next_mcuposn(j, rsti, p); };
        while (true) {
            int lastdc[4] = {0, 0, 0, 0};
            int sta = 0;
            p.rstw = rsti;
            pw.eobrun = 0;
            if (j.jpegtype == 1) {
                // ---- sequential scan
                while (sta == 0) {
                    encode_block_seq(bw, planes[p.cmp] + (size_t)p.dpos * 64, t.dc[t.td[p.cmp]], t.ac[t.ta[p.cmp]], lastdc[p.cmp]);
                    sta = next_pos();
                }
            } else if (inter || sc.to == 0) {
                if (sc.sah == 0) {
                    // ---- DC first stage
                    while (sta == 0) {
                        const HuffTable& dct = t.dc[t.td[p.cmp]];
                        const int tmp = coef(0) >> sc.sal;
                        const int16_t diff = (int16_t)(tmp - lastdc[p.cmp]);
                        lastdc[p.cmp] = tmp;
                        const int s = bitlen16(diff > 0 ? diff : -diff);
                        const int nb = diff > 0 ? diff : (diff - 1) + (1 << s);
                        bw.put(dct.ecode[s], dct.elen[s]);
                        bw.put((uint32_t)nb, s);
                        sta = next_pos();
                    }
                } else {
                    // ---- DC refinement bit
                    while (sta == 0) {
                        bw.put((uint32_t)((coef(0) >> sc.sal) & 1), 1);
                        sta = next_pos();
                    }
                }
            } else if (sc.sah == 0) {
                // ---- AC first stage
                const HuffTable& act = t.ac[t.ta[p.cmp]];
                const uint64_t band = (sc.to == 63 ? ~0ull : (1ull << (sc.to + 1)) - 1) & ~((1ull << sc.from) - 1);
                while (sta == 0) {
                    uint64_t m = magnitude_mask_zigzag(planes[p.cmp] + (size_t)p.dpos * 64, 1 << sc.sal) & band;
                    int prev = sc.from - 1;
                    if (m) pw.flush_eobrun(act);
                    while (m) {
                        const int bpos = __builtin_ctzll(m);
                        m &= m - 1;
                        int z = bpos - prev - 1;
                        prev = bpos;
                        const int tmp = fdiv2(coef(bpos), sc.sal);
                        while (z >= 16) { bw.put(act.ecode[0xF0], act.elen[0xF0]); z -= 16; }
                        const int a = tmp > 0 ? tmp : -tmp;
                        const int s = bitlen16(a);
                        const int nb = tmp > 0 ? tmp : (tmp - 1) + (1 << s);
                        const int hc = (z << 4) + s;
                        bw.put(act.ecode[hc], act.elen[hc]);
                        bw.put((uint32_t)nb, s);
                    }
                    if (prev < sc.to) {
                        ++pw.eobrun;
                        if (pw.eobrun == (unsigned)act.max_eobrun) pw.flush_eobrun(act);
                    }
                    sta = next_pos();
                }
                pw.flush_eobrun(act);
            } else {
                // ---- AC refinement
                const HuffTable& act = t.ac[t.ta[p.cmp]];
                const uint64_t band = (sc.to == 63 ? ~0ull : (1ull << (sc.to + 1)) - 1) & ~((1ull << sc.from) - 1);
                while (sta == 0) {
                    // sig: non-zero at this bit plane; old: significant before this scan (|v| >> sal >= 2);
                    // the remaining sig positions turn significant here (|v| >> sal == 1)
                    const int16_t* blkp = planes[p.cmp] + (size_t)p.dpos * 64;
                    uint64_t sig = magnitude_mask_zigzag(blkp, 1 << sc.sal) & band;
                    const uint64_t old = magnitude_mask_zigzag(blkp, 2 << sc.sal) & band;
                    const uint64_t fresh = sig & ~old;
                    const int eob = fresh ? 64 - __builtin_clzll(fresh) : sc.from;
                    if (eob > sc.from && pw.eobrun > 0) { pw.flush_eobrun(act); pw.flush_crbits(); }
                    int z = 0, prev = sc.from - 1;
                    while (sig) {
                        const int bpos = __builtin_ctzll(sig);
                        sig &= sig - 1;
                        const int v = coef(bpos);
                        if (bpos >= eob) {                 // behind the last new coefficient: correction bits only
                            pw.push_crbit((uint32_t)(((v < 0 ? -v : v) >> sc.sal) & 1));
                            continue;
                        }
                        z += bpos - prev - 1;
                        prev = bpos;
                        while (z >= 16) { bw.put(act.ecode[0xF0], act.elen[0xF0]); pw.flush_crbits(); z -= 16; }
                        if ((fresh >> bpos) & 1) {
                            const int hc = (z << 4) + 1;
                            bw.put(act.ecode[hc], act.elen[hc]);
                            bw.put(v > 0 ? 1u : 0u, 1);
                            pw.flush_crbits();
                            z = 0;
                        } else {
                            pw.push_crbit((uint32_t)(((v < 0 ? -v : v) >> sc.sal) & 1));
                        }
                    }
                    if (eob <= sc.to) {
                        ++pw.eobrun;
                        if (pw.eobrun == (unsigned)act.max_eobrun) { pw.flush_eobrun(act); pw.flush_crbits(); }
                    }
                    sta = next_pos();
                }
                pw.flush_eobrun(act);
                pw.flush_crbits();
            }
            bw.pad((uint8_t)j.padbit);
            if (sta == 2) break;
            // restart: marker after the padded byte when the scan's marker budget allows (:2640-2650)
            if (rsti > 0) {
                if (rst_ok()) {
                    bw.raw(0xFF);
                    bw.raw((uint8_t)(0xD0 + (cpos & 7)));
                    ++cpos; ++rst_this_scan;
                } else {
                    rst_stuck = true;
                }
            }
        }
        // bogus trailing restart markers of this scan (:2711-2719)
        if ((size_t)scan - 1 < j.rst_err.size())
            for (unsigned i = 0; i < j.rst_err[scan - 1]; ++i) { bw.raw(0xFF); bw.raw((uint8_t)(0xD0 + (cpos & 7))); ++cpos; }
    }
    bw.finish();
    if (scan == 0) { err = "no scan found"; return false; }
    if (pw.bad) { err = "coefficients not expressible with the scan's huffman tables"; return false; }
    if (lf.jpeg_size >= j.grb.size() && out.size() > lf.jpeg_size - j.grb.size()) out.resize(lf.jpeg_size - j.grb.size());
    out.insert(out.end(), j.grb.begin(), j.grb.end());
    return size_checks(lf, out.size() + j.prefix.size(), err);
}

}  // namespace lephost
