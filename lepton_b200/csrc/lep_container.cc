// lep_container.cc -- .lep container writer/reader: thread-segment selection, ThreadHandoff wire form,
// MuxWriter packetisation, fixed header + zlib'd JPEG header blob, size trailer.
//
// Byte-exact restatement of write_ujpg (jpgcoder.cc:3779-4097), ThreadHandoff::serialize
// (thread_handoff.cc:46-76), MuxWriter (src/io/MuxReader.hh:336-522) and the stream interleave + trailer of
// vp8_full_encoder (src/lepton/vp8_encoder.cc:573-614) for the reference's options that keep version 1 / zlib
// header and up to 8 threads (no -startbyte/-trunc slices).
#include <zlib.h>

#include <algorithm>
#include <cstring>

#include "lep_host.h"

namespace lephost {

namespace {
inline void le32(std::vector<uint8_t>& v, uint32_t x) { for (int i = 0; i < 4; ++i) v.push_back((uint8_t)(x >> (8 * i))); }
inline void put(std::vector<uint8_t>& v, const char* s, size_t n) { v.insert(v.end(), s, s + n); }
}  // namespace

// ------------------------------------------------------------------------------------------------
// write_ujpg thread-segment selection (jpgcoder.cc:3860-3934): NUM_THREADS = min(MAX_NUM_THREADS = 8,
// -maxencodethreads) (:2196, :3862), min_encode_threads from -minencodethreads (default 1), -evensplit = rows divided evenly instead of bytes.
// ------------------------------------------------------------------------------------------------
Splits select_splits(const Jpeg& j, unsigned max_threads, unsigned min_threads, bool even_split) {
    const std::vector<Handoff>& rows = j.rows;
    Splits sp;
    const uint32_t byte_size = rows.back().segment_size - rows.front().segment_size;
    const uint32_t num_rows = (uint32_t)rows.size();
    unsigned nthreads = std::min(8u, std::max(1u, max_threads));
    min_threads = std::min(std::max(min_threads, 1u), 8u);
    if (num_rows / 2 < nthreads) {
        unsigned desired = std::max(num_rows / 2, min_threads);
        nthreads = std::min(std::max(desired, 1u), nthreads);
    }
    if (byte_size < 125000) nthreads = std::min(std::max(min_threads, 1u), nthreads);
    else if (byte_size < 250000) nthreads = std::min(std::max(min_threads, 2u), nthreads);
    else if (byte_size < 500000) nthreads = std::min(std::max(min_threads, 4u), nthreads);

    std::vector<int> idx(nthreads, 0);
    for (unsigned i = 0; !even_split && i + 1 < nthreads; ++i) {
        uint32_t desired = rows.back().segment_size;
        desired -= rows.front().segment_size;
        desired *= (i + 1);
        desired /= nthreads;
        desired += rows.front().segment_size;
        auto split = std::lower_bound(rows.begin() + 1, rows.end(), desired,
                                      [](const Handoff& a, uint32_t b) { return a.segment_size < b; });
        if (split == rows.begin() && split != rows.end()) {
        } else if (split != rows.begin() + 1) {
            --split;
        }
        idx[i] = (int)(split - rows.begin());
    }
    for (unsigned i = 0; even_split && i + 1 < nthreads; ++i) idx[i] = (int)(rows.size() * (i + 1) / nthreads);   // -evensplit (:3898-3900)
    for (unsigned k = 0; k + 1 < nthreads; ++k) {
        if (idx[k] == idx[k + 1]) {      // note: compares against the still-zero last entry for k == nthreads-2, as the reference does
            for (unsigned i = 0; i + 1 < nthreads; ++i) idx[i] = (int)((i + 1) * rows.size() / nthreads);
            break;
        }
    }
    idx[nthreads - 1] = (int)rows.size() - 1;
    size_t last = 0;
    for (unsigned i = 0; i < nthreads; ++i) {
        const size_t b = last, e = (size_t)idx[i];
        last = e;
        Handoff h = rows[b];                      // ThreadHandoff::operator- (thread_handoff.cc:100-106)
        h.luma_y_end = rows[e].luma_y_start;
        h.segment_size = rows[e].segment_size - rows[b].segment_size;
        if (i + 1 == nthreads && rows[e].num_overhang_bits) ++h.segment_size;
        sp.selected.push_back(h);
    }
    return sp;
}

// ------------------------------------------------------------------------------------------------
// MuxWriter (src/io/MuxReader.hh:336-522), version 1 (no EOF marker)
// ------------------------------------------------------------------------------------------------
// The writer's decisions -- when a stream is flushed, as packets of which kind -- depend only on how many bytes each
// stream has been given so far, never on the bytes.  So the writer is kept data-free: it is driven with lengths and
// emits the packet list (stream id, header bytes, offset and length inside the stream); mux_streams copies by that
// list on the host, the device gather kernel (lep_capi.cu, lepb200_encode_fetch_files) by the same list on the GPU.
namespace {
struct Mux {
    enum { NS = 16, MAX_BUFFER_LAG = 65537 };
    std::vector<MuxPacket>& out;
    uint32_t pending[NS];            // bytes written to the stream's buffer and not yet flushed
    uint32_t consumed[NS];           // offset inside the stream of the first pending byte
    uint32_t flushed[NS], low_water[NS];
    bool opened[NS];
    uint32_t total_written = 0;
    explicit Mux(std::vector<MuxPacket>& o) : out(o) { for (int i = 0; i < NS; ++i) { pending[i] = consumed[i] = flushed[i] = low_water[i] = 0; opened[i] = false; } }

    static uint32_t high_water(uint32_t f) { return (f & 0xffffc000u) ? 65536 : ((f & 0xfffff000u) ? 16384 : 4096); }

    void emit(int id, uint8_t nhdr, uint8_t h0, uint8_t h1, uint8_t h2, uint32_t len) {
        MuxPacket p;
        p.id = (uint8_t)id; p.nhdr = nhdr; p.hdr[0] = h0; p.hdr[1] = h1; p.hdr[2] = h2;
        p.src_off = consumed[id]; p.len = len;
        out.push_back(p);
        consumed[id] += len; pending[id] -= len;
        total_written += len; flushed[id] += len;
    }
    void flush_full(int id, uint32_t n) {
        if (!n) return;
        do {
            const uint32_t w = std::min(n, 65536u);
            emit(id, 3, (uint8_t)id, (uint8_t)((w - 1) & 0xff), (uint8_t)(((w - 1) >> 8) & 0xff), w);
            n -= w;
        } while (n > 0);
        low_water[id] = total_written;
    }
    void flush_partial(int id, uint32_t n) {
        uint8_t code = (uint8_t)id;
        uint32_t len;
        if (n < 4096) { flush_full(id, n); return; }
        if (n < 16384) { if (n > 8192) { flush_full(id, n); return; } len = 4096; code |= 1 << 4; }
        else if (n < 65536) { if (n > 32768) { flush_full(id, n); return; } len = 16384; code |= 2 << 4; }
        else { if (n > 131072) { flush_full(id, n); return; } len = 65536; code |= 3 << 4; }
        for (uint32_t w = 0; w + len <= n; w += len) {
            if (pending[id] == 0) continue;
            emit(id, 1, code, 0, 0, len);
        }
        const uint32_t delta = pending[id];
        low_water[id] = delta > total_written ? 0 : total_written - delta;
    }
    void flush(int id) {
        for (int i = 0; i < NS; ++i) {
            const uint32_t n = pending[i];
            if (i == id || !n) continue;
            const bool urgent = total_written - low_water[i] > MAX_BUFFER_LAG;
            if (n < 4096) { if (urgent) flush_full(i, n); }
            else if (urgent && n < 16384) flush_full(i, n);
            else flush_partial(i, n);
        }
        flush_partial(id, pending[id]);
    }
    void write(int id, uint32_t n) {
        opened[id] = true;
        pending[id] += n;
        if (pending[id] >= high_water(flushed[id])) flush(id);
    }
    void close() {
        for (int i = 0; i < NS; ++i)
            if (pending[i]) flush_full(i, pending[i]);
    }
};
}  // namespace

void plan_mux(const size_t* lens, int nseg, std::vector<MuxPacket>& out) {
    // interleave schedule of vp8_full_encoder (vp8_encoder.cc:575-594): 256 bytes, then 4096, then 65536 per turn
    out.clear();
    Mux mux(out);
    std::vector<size_t> done((size_t)std::max(nseg, 0), 0);
    bool any = true;
    while (any) {
        any = false;
        for (int i = 0; i < nseg && i < 16; ++i) {
            if (lens[i] > done[i]) {
                any = true;
                size_t maxw = 65536;
                if (done[i] == 0) maxw = 256;
                else if (done[i] == 256) maxw = 4096;
                const size_t w = std::min(maxw, lens[i] - done[i]);
                mux.write(i, (uint32_t)w);
                done[i] += w;
            }
        }
    }
    mux.close();
}

void mux_streams(const std::vector<std::pair<const uint8_t*, size_t>>& streams, std::vector<uint8_t>& out) {
    std::vector<size_t> lens(streams.size());
    for (size_t i = 0; i < streams.size(); ++i) lens[i] = streams[i].second;
    std::vector<MuxPacket> plan;
    plan_mux(lens.data(), (int)streams.size(), plan);
    for (const MuxPacket& p : plan) {
        out.insert(out.end(), p.hdr, p.hdr + p.nhdr);
        out.insert(out.end(), streams[p.id].first + p.src_off, streams[p.id].first + p.src_off + p.len);
    }
}

// ------------------------------------------------------------------------------------------------
// write_ujpg header + trailer
// ------------------------------------------------------------------------------------------------
namespace {
// zlib level 9, deflate(Z_NO_FLUSH) then Z_FINISH (src/io/ZlibCompression.cc:44-75)
bool deflate9(const std::vector<uint8_t>& blob, std::vector<uint8_t>& z, std::string& err) {
    z.resize(compressBound((uLong)blob.size()));
    z_stream strm;
    memset(&strm, 0, sizeof(strm));
    if (deflateInit(&strm, 9) != Z_OK) { err = "deflateInit failed"; return false; }
    strm.next_in = const_cast<uint8_t*>(blob.data()); strm.avail_in = (uInt)blob.size();
    strm.next_out = z.data(); strm.avail_out = (uInt)z.size();
    int ret = deflate(&strm, Z_NO_FLUSH);
    while (ret != Z_STREAM_END) {
        ret = deflate(&strm, Z_FINISH);
        if (ret != Z_OK && ret != Z_STREAM_END && ret != Z_BUF_ERROR) { deflateEnd(&strm); err = "deflate failed"; return false; }
    }
    z.resize(z.size() - strm.avail_out);
    deflateEnd(&strm);
    return true;
}

// the 28 fixed bytes (lepton_header, jpgcoder.cc:551; :4044-4066), the zlib'd blob and "CMP"
void fixed_header(uint8_t flag, uint8_t nseg, uint32_t filesize, const std::vector<uint8_t>& z, std::vector<uint8_t>& out) {
    out.clear();
    out.reserve(28 + z.size() + 3);
    out.push_back(0xCF); out.push_back(0x84);
    out.push_back(1);                                      // ujgversion
    out.push_back(flag);
    out.push_back(nseg);
    out.push_back(0); out.push_back(0); out.push_back(0);
    for (int i = 0; i < 12; ++i) out.push_back(0);         // GIT_REVISION "" (:4058-4060)
    le32(out, filesize);
    le32(out, (uint32_t)z.size());
    out.insert(out.end(), z.begin(), z.end());
    put(out, "CMP", 3);
}

void put_handoffs(std::vector<uint8_t>& blob, const std::vector<Handoff>& hs) {
    blob.push_back('H');                                   // luma_mrk (jpgcoder.cc:3970)
    blob.push_back('H');                                   // ThreadHandoff::serialize (thread_handoff.cc:46-76)
    blob.push_back((uint8_t)hs.size());
    for (const Handoff& h : hs) {
        blob.push_back(h.luma_y_start & 255); blob.push_back(h.luma_y_start >> 8);
        le32(blob, h.segment_size);
        blob.push_back(h.overhang_byte);
        blob.push_back(h.num_overhang_bits);
        for (int i = 0; i < 3; ++i) { uint16_t dc = (uint16_t)h.last_dc[i]; blob.push_back(dc & 255); blob.push_back(dc >> 8); }
        blob.push_back(0); blob.push_back(0);
    }
}
}  // namespace

bool build_lep_header(const Jpeg& j, const Splits& sp, std::vector<uint8_t>& out, std::string& err) {
    std::vector<uint8_t> blob;
    blob.reserve(j.hdr.size() + j.prefix.size() + j.grb.size() + 512);
    put(blob, "HDR", 3);
    le32(blob, (uint32_t)j.hdr.size());
    blob.insert(blob.end(), j.hdr.begin(), j.hdr.end());
    put(blob, "P0D", 3);
    blob.push_back((uint8_t)j.padbit);
    put_handoffs(blob, sp.selected);
    if (!j.rst_cnt.empty()) {
        put(blob, "CRS", 3);
        le32(blob, (uint32_t)j.rst_cnt.size());
        for (uint32_t c : j.rst_cnt) le32(blob, c);
    }
    if (!j.rst_err.empty()) {
        put(blob, "FRS", 3);
        le32(blob, (uint32_t)j.rst_err.size());
        blob.insert(blob.end(), j.rst_err.begin(), j.rst_err.end());
    }
    if (j.early_eof) {                                     // jpgcoder.cc:3996-4007
        put(blob, "EEE", 3);
        le32(blob, (uint32_t)j.max_cmp); le32(blob, (uint32_t)j.max_bpos); le32(blob, (uint32_t)j.max_sah);
        for (int i = 0; i < 4; ++i) le32(blob, (uint32_t)j.max_dpos[i]);
    }
    if (!j.prefix.empty()) {                               // -embedding=N: the bytes in front of the SOI (jpgcoder.cc:4009-4017)
        put(blob, "PGE", 3);
        le32(blob, (uint32_t)j.prefix.size());
        blob.insert(blob.end(), j.prefix.begin(), j.prefix.end());
    }
    if (!j.grb.empty()) {
        put(blob, "GRB", 3);
        le32(blob, (uint32_t)j.grb.size());
        blob.insert(blob.end(), j.grb.begin(), j.grb.end());
    }
    std::vector<uint8_t> z;
    if (!deflate9(blob, z, err)) return false;
    // 'Z': g_allow_progressive cleared for baseline files (:3298-3300, :4044-4052)
    fixed_header(j.is_baseline ? 'Z' : 'X', (uint8_t)sp.selected.size(), j.filesize, z, out);
    return true;
}

// ------------------------------------------------------------------------------------------------
// The generic container of -permissive (generic_compress.cc:60-200)
// ------------------------------------------------------------------------------------------------
const std::vector<uint8_t>& generic_jpeg_header() {
    // A 1x1 greyscale baseline JPEG, every segment after its SOI up to and including the SOS, then two bytes of scan:
    // JFIF APP0 (version 1.1, 28 x 28 dots per cm, no thumbnail); the luminance table of ITU-T T.81 Annex K.1 scaled as
    // libjpeg does for quality 92 ((q * 16 + 50) / 100), in zig-zag order; SOF0 8-bit 1x1, one component (id 1, 1x1,
    // table 0); one DC and one AC table that each hold a single 1-bit code (DC category 9, AC end-of-block); the SOS.
    static const std::vector<uint8_t> hdr = [] {
        static const uint8_t annex_k1[64] = {
            16, 11, 10, 16, 24, 40, 51, 61,    12, 12, 14, 19, 26, 58, 60, 55,
            14, 13, 16, 24, 40, 57, 69, 56,    14, 17, 22, 29, 51, 87, 80, 62,
            18, 22, 37, 56, 68, 109, 103, 77,  24, 35, 55, 64, 81, 104, 113, 92,
            49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
        std::vector<uint8_t> h = {0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x02, 0x00, 0x1C, 0x00, 0x1C, 0x00, 0x00,
                                  0xFF, 0xDB, 0x00, 0x43, 0x00};
        // zig-zag order: anti-diagonal d = row + col, walked upwards for even d and downwards for odd d
        for (int d = 0; d < 15; ++d) {
            const int lo = std::max(0, d - 7), hi = std::min(d, 7);
            for (int k = 0; k <= hi - lo; ++k) {
                const int row = (d & 1) ? lo + k : hi - k;
                h.push_back((uint8_t)std::max(1, std::min(255, (annex_k1[row * 8 + d - row] * 16 + 50) / 100)));
            }
        }
        const uint8_t rest[] = {0xFF, 0xC0, 0x00, 0x0B, 0x08, 0x00, 0x01, 0x00, 0x01, 0x01, 0x01, 0x11, 0x00,
                                0xFF, 0xC4, 0x00, 0x14, 0x00, 0x01, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x09,
                                0xFF, 0xC4, 0x00, 0x14, 0x10, 0x01, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0x00,
                                0xFF, 0xDA, 0x00, 0x08, 0x01, 0x01, 0x00, 0x00, 0x3F, 0x00, 0x54, 0xDD};
        h.insert(h.end(), rest, rest + sizeof(rest));
        return h;
    }();
    return hdr;
}

bool write_generic_lep(const uint8_t* data, size_t n, std::vector<uint8_t>& out, std::string& err) {
    out.clear();
    if (n == 0) { err = "empty input"; return false; }                  // UNSUPPORTED_JPEG in the reference
    if (n > 0xFFFFFFFFu - 4096) { err = "input too large for the container's size fields"; return false; }
    const std::vector<uint8_t>& hdr = generic_jpeg_header();
    std::vector<uint8_t> blob;
    blob.reserve(hdr.size() + n + 256);
    put(blob, "HDR", 3);
    le32(blob, (uint32_t)hdr.size());
    blob.insert(blob.end(), hdr.begin(), hdr.end());
    put(blob, "P0D", 3);
    blob.push_back(0);
    put_handoffs(blob, std::vector<Handoff>(GENERIC_SEGMENTS));   // MAX_NUM_THREADS zeroed handoffs
    put(blob, "PGE", 3);                                   // the whole input, restored in front of nothing
    le32(blob, (uint32_t)n);
    blob.insert(blob.end(), data, data + n);
    put(blob, "GRB", 3);                                   // and an empty trailer
    le32(blob, 0);
    std::vector<uint8_t> z;
    if (!deflate9(blob, z, err)) return false;
    fixed_header('Y', (uint8_t)GENERIC_SEGMENTS, (uint32_t)n, z, out);
    le32(out, (uint32_t)out.size() + 4);                   // no mux packets: the size trailer follows "CMP"
    return true;
}

bool write_lep(const Jpeg& j, const Splits& sp, const std::vector<std::pair<const uint8_t*, size_t>>& streams,
               std::vector<uint8_t>& out, std::string& err) {
    std::vector<uint8_t> hdr;
    if (!build_lep_header(j, sp, hdr, err)) return false;
    size_t total_stream = 0;
    for (auto& s : streams) total_stream += s.second;
    out.clear();
    out.reserve(hdr.size() + total_stream + total_stream / 1024 + 64);
    out.insert(out.end(), hdr.begin(), hdr.end());
    mux_streams(streams, out);
    le32(out, (uint32_t)out.size() + 4);                   // vp8_encoder.cc:603-614
    return true;
}

}  // namespace lephost
