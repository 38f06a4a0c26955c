// lep_file.cc -- file-level drop-in: JPEG bytes -> .lep bytes and back, batched.
//
// Host threads do what the reference's jpgcoder.cc does around the codec boundary (read_jpeg / write_ujpg on the way in,
// read_ujpg on the way out, plus decode_jpeg / recode_*_jpeg for the files the GPU Huffman kernels do not take:
// progressive, truncated, several scans); Huffman decode / encode of complete baseline scans and the arithmetic coding
// go through the C ABI of lep_capi.cu to the sm_90a kernels.  No CPU arithmetic coder exists in this library.
#include <atomic>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <memory>
#include <condition_variable>
#include <mutex>
#include <thread>
#include <array>
#include <algorithm>
#include <ctime>
#include <string>
#include <vector>

#include <cuda_runtime.h>

#include "../../include/lepton_b200.h"
#include "lep_host.h"

using namespace lephost;

struct lepb200_codec {
    lepb200_ctx* ctx = nullptr;     // == ctx2[0]
    static constexpr int NCTX = 4;
    lepb200_ctx* ctx2[NCTX] = {nullptr, nullptr, nullptr, nullptr};   // one context (stream, device arenas) per chunk in flight
    int concurrent = 4;             // chunks of one call that run at the same time (LEPB200_CHUNKS_IN_FLIGHT), 1..NCTX
    int nthreads = 1;
    int chunk_images = 4096;
    size_t plane_cap = size_t(14) << 30;   // coefficient-plane bytes of the chunks in flight, divided among them; set to 18 % of the
                                           // device memory at creation: the arenas of a chunk (planes, tokens, streams, models, each with
                                           // 1/8 headroom) take about three times its plane bytes, plus 5.6 GB of encode models per context
    int arena_dir[NCTX] = {0, 0, 0, 0};    // direction of the call each context's arenas were sized for: 1 compress, 2 decompress
    bool gpu_huffman = true;       // Huffman-decode eligible chunks on the GPU (SURVEY 8(f) row 1)
    bool even_split = false;       // -evensplit (jpgcoder.cc:1063-1064)
    unsigned max_encode_threads = 8, min_encode_threads = 1;   // -maxencodethreads= / -minencodethreads= (jpgcoder.cc:1080-1089)
    bool verify = false;           // -verify: decode every .lep again and compare with the input before handing it out
    bool allow_progressive = true; // false: -rejectprogressive (files that are not single-scan-interleaved baseline exit with code 8)
    bool zlib0 = false;            // -zlib0: restored JPEGs are handed out as zlib streams of stored blocks
    long long embedding = -1;      // -embedding=N (>= 0): every input is a JPEG whose SOI sits at byte N; the bytes in front are kept
    bool discard_meta = false;     // -d: the container keeps only the header segments the coefficients are coded with
    void* arena[4] = {nullptr, nullptr, nullptr, nullptr};  // pinned host memory for coefficient planes, one per in-flight chunk
    size_t arena_cap[4] = {0, 0, 0, 0};
    std::vector<std::vector<uint8_t>> outputs;
    std::vector<std::vector<uint8_t>> joined;   // decompress: inputs of several members, their restored members concatenated
    std::string err;
    // timing of the last call (seconds): parse+huffman, gpu (upload+kernel+fetch), container
    double t_front = 0, t_gpu = 0, t_back = 0, t_huff_ms = 0;
    std::atomic<int> n_gpu_recoded{0};   // files of the last decompress call whose scan was Huffman-encoded on the device
};

namespace {

template <class F>
void parallel_for(int n, int nthreads, F&& f) {
    nthreads = std::max(1, std::min(nthreads, n));
    if (nthreads == 1) { for (int i = 0; i < n; ++i) f(i); return; }
    std::atomic<int> next(0);
    std::vector<std::thread> th;
    th.reserve(nthreads);
    for (int t = 0; t < nthreads; ++t)
        th.emplace_back([&]() { for (int i; (i = next.fetch_add(1)) < n;) f(i); });
    for (auto& t : th) t.join();
}

double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return ts.tv_sec + 1e-9 * ts.tv_nsec;
}

bool reserve_arena(lepb200_codec* c, int slot, size_t bytes) {
    if (bytes <= c->arena_cap[slot]) return true;
    if (c->arena[slot]) lepb200_pinned_free(c->arena[slot]);
    c->arena[slot] = nullptr; c->arena_cap[slot] = 0;
    size_t want = bytes + bytes / 8 + 4096;
    c->arena[slot] = lepb200_pinned_alloc(want);
    if (!c->arena[slot]) return false;
    c->arena_cap[slot] = want;
    return true;
}

void fill_image(lepb200_image& im, const Jpeg& j, int16_t* const planes[4], const std::vector<Handoff>& sel) {
    memset(&im, 0, sizeof(im));
    im.ncmp = j.ncmp; im.mcuv = j.mcuv;
    for (int c = 0; c < j.ncmp; ++c) {
        im.bch[c] = j.cmp[c].bch; im.bcv[c] = j.cmp[c].bcv;
        im.trunc_bcv[c] = j.trunc_bcv[c] ? j.trunc_bcv[c] : j.cmp[c].bcv;
        im.trunc_bc[c] = j.trunc_bc[c] ? j.trunc_bc[c] : j.cmp[c].bc;
        memcpy(im.qtable_zigzag[c], j.qtables[j.cmp[c].tq], 128);
        im.planes[c] = planes[c];
    }
    im.nseg = (int)sel.size();
    for (size_t s = 0; s < sel.size(); ++s) im.luma_y_start[s] = sel[s].luma_y_start;
}

}  // namespace

// A context keeps its device arenas only while calls of the same direction use it: the arenas of the other direction, and
// those of contexts a call leaves idle, would otherwise stay reserved next to the ones the call grows.
static void keep_arenas_for(lepb200_codec* c, int dir, int used) {
    for (int s = 0; s < lepb200_codec::NCTX; ++s) {
        const int want = s < used ? dir : 0;
        if (c->arena_dir[s] && c->arena_dir[s] != want) lepb200_release_device_buffers(c->ctx2[s]);
        c->arena_dir[s] = want;
    }
}

extern "C" {

int lepb200_codec_create(lepb200_codec** out, int device, int host_threads) {
    if (!out) return LEPB200_ERR_INVALID;
    *out = nullptr;
    lepb200_ctx* ctx = nullptr;
    int r = lepb200_create(&ctx, device);
    if (r) return r;
    lepb200_codec* c = new lepb200_codec();
    c->ctx = ctx;
    c->ctx2[0] = ctx;
    for (int s = 1; s < lepb200_codec::NCTX; ++s) {
        r = lepb200_create(&c->ctx2[s], device);
        if (r) { for (int q = 0; q < s; ++q) lepb200_destroy(c->ctx2[q]); delete c; return r; }
    }
    c->nthreads = host_threads > 0 ? host_threads : (int)std::max(1u, std::thread::hardware_concurrency());
    size_t free_bytes = 0, total_bytes = 0;
    if (cudaMemGetInfo(&free_bytes, &total_bytes) == cudaSuccess && total_bytes) c->plane_cap = total_bytes / 100 * 18;
    for (int s = 0; s < lepb200_codec::NCTX; ++s) lepb200_set_host_threads(c->ctx2[s], c->nthreads);
    if (const char* e = getenv("LEPB200_CHUNKS_IN_FLIGHT")) c->concurrent = std::min((int)lepb200_codec::NCTX, std::max(1, atoi(e)));
    *out = c;
    return LEPB200_OK;
}

void lepb200_codec_destroy(lepb200_codec* c) {
    if (!c) return;
    for (int s = 0; s < 4; ++s) if (c->arena[s]) lepb200_pinned_free(c->arena[s]);
    for (int s = 0; s < lepb200_codec::NCTX; ++s) lepb200_destroy(c->ctx2[s]);
    delete c;
}

const char* lepb200_codec_last_error(const lepb200_codec* c) {
    if (!c) return "null codec";
    return c->err.empty() ? lepb200_last_error(c->ctx) : c->err.c_str();
}

lepb200_ctx* lepb200_codec_ctx(lepb200_codec* c) { return c ? c->ctx : nullptr; }
uint64_t lepb200_codec_kernel_launches(const lepb200_codec* c) {
    uint64_t n = 0;
    for (int s = 0; c && s < lepb200_codec::NCTX; ++s) n += lepb200_kernel_launches(c->ctx2[s]);
    return n;
}
void lepb200_codec_set_chunk_images(lepb200_codec* c, int n) { if (c && n > 0) c->chunk_images = n; }
void lepb200_codec_set_gpu_huffman(lepb200_codec* c, int on) { if (c) c->gpu_huffman = on != 0; }
void lepb200_codec_set_allow_progressive(lepb200_codec* c, int on) { if (c) c->allow_progressive = on != 0; }
void lepb200_codec_set_even_split(lepb200_codec* c, int on) { if (c) c->even_split = on != 0; }
void lepb200_codec_set_verify(lepb200_codec* c, int on) { if (c) c->verify = on != 0; }
void lepb200_codec_set_zlib0(lepb200_codec* c, int on) { if (c) c->zlib0 = on != 0; }
void lepb200_codec_set_embedding(lepb200_codec* c, long long offset) { if (c) c->embedding = offset < 0 ? -1 : offset; }
void lepb200_codec_set_discard_meta(lepb200_codec* c, int on) { if (c) c->discard_meta = on != 0; }
void lepb200_codec_set_encode_threads(lepb200_codec* c, int min_threads, int max_threads) {
    if (!c) return;
    c->min_encode_threads = (unsigned)std::min(std::max(min_threads, 1), 8);
    c->max_encode_threads = (unsigned)std::min(std::max(max_threads, 1), 8);
}
double lepb200_codec_last_huffman_ms(const lepb200_codec* c) { return c ? c->t_huff_ms : -1.0; }
int lepb200_codec_last_gpu_recoded(const lepb200_codec* c) { return c ? c->n_gpu_recoded.load() : 0; }

void lepb200_codec_last_timing(const lepb200_codec* c, double* front_s, double* gpu_s, double* back_s) {
    if (!c) return;
    if (front_s) *front_s = c->t_front;
    if (gpu_s) *gpu_s = c->t_gpu;
    if (back_s) *back_s = c->t_back;
}

// JPEG files -> .lep files.  out[i].data points into codec-owned memory, valid until the next call.
//
// The batch is cut into LARGE chunks (up to `chunk_images` files and `plane_cap` bytes of coefficient planes): the
// Huffman-decode and range-coder kernels are latency-bound chains whose duration hardly depends on how many images they
// cover, so a launch should cover as many as device memory allows.  Chunks run through a 3-stage lock-step pipeline on
// two alternating contexts:
//   front (host threads) parse + de-stuff every file straight into the context's pinned staging buffer; files the GPU
//                        Huffman decoder cannot take (progressive, truncated, several scans) are Huffman-decoded here
//                        into a pinned plane arena instead
//   gpu                  H2D -> Huffman kernel -> thread-segment selection (host) -> token pre-pass -> kernel A ->
//                        kernel B -> compaction -> D2H
//   back  (host threads) mux + container of every file
namespace {

struct ChunkState {
    int begin = 0, end = 0;
    std::vector<std::unique_ptr<Jpeg>> js;              // per file of the chunk
    std::vector<std::array<int16_t*, 4>> planes;        // host planes of host-decoded files (else null)
    std::vector<Splits> splits;
    std::vector<uint8_t> host_decoded;                  // 1: planes came from the host Huffman decoder
    std::vector<lepb200_image> imgs;                    // batch order == idx order
    std::vector<int> idx;                               // file index (relative to begin) of imgs[q]
    std::vector<int> seg_base;
    std::vector<lepb200_stream> streams;
    std::vector<lepb200_jpeg_scan> scans;               // per batch image
    std::vector<std::vector<lepb200_huffrow>> rowbuf;
    int gpu_rc = 0;
    bool any_gpu_huffman = false;
    std::vector<std::vector<uint8_t>> headers;   // device container assembly: per batch image everything in front of the mux packets
    std::vector<lepb200_result> files;           // ... and the finished files (pinned memory of the chunk's context)
};

// The device Huffman decoder's job for one JPEG (sc.rows stays the caller's): geometry, and with a set-up the entropy bytes,
// restart interval and tables; without one a placeholder that only gets its plane slot.
void fill_jpeg_scan(const Jpeg& j, const GpuScanSetup* gs, lepb200_jpeg_scan& sc) {
    lepb200_huffrow* rows = sc.rows;
    memset(&sc, 0, sizeof(sc));
    sc.rows = rows;
    sc.ncmp = j.ncmp; sc.mcuh = j.mcuh; sc.mcuv = j.mcuv;
    for (int t = 0; t < j.ncmp && t < 3; ++t) { sc.H[t] = j.cmp[t].H; sc.V[t] = j.cmp[t].V; sc.nch[t] = j.cmp[t].nch; sc.ncv[t] = j.cmp[t].ncv; }
    if (!gs) return;
    sc.entropy = j.huff.data(); sc.nbytes = (uint32_t)j.huff.size(); sc.rsti = gs->rsti;
    for (int t = 0; t < j.ncmp; ++t) { sc.dc[t] = gs->dc[t]; sc.ac[t] = gs->ac[t]; }
}

}  // namespace

int lepb200_compress_jpegs(lepb200_codec* c, const lepb200_buffer* jpegs, int n, lepb200_result* out) {
    if (!c || !jpegs || !out || n <= 0) return LEPB200_ERR_INVALID;
    const bool trace = getenv("LEPB200_TRACE") != nullptr;           // stage timeline on stderr (diagnostics)
    const double t_origin = now_s();
    auto mark = [&](const char* what, int k, double t_begin) {
        if (trace) fprintf(stderr, "[trace] %-16s chunk %d  %8.1f -> %8.1f ms\n", what, k, (t_begin - t_origin) * 1e3, (now_s() - t_origin) * 1e3);
    };
    c->err.clear();
    c->t_front = c->t_gpu = c->t_back = 0;
    // ---- chunk boundaries
    std::vector<size_t> need(n);
    parallel_for(n, c->nthreads, [&](int i) { need[i] = peek_plane_bytes(jpegs[i].data, jpegs[i].len, c->embedding); });
    // Chunks: up to `concurrent` of them run at the same time, each on its own context (stream + device arenas), so
    // that the latency-bound kernels of one chunk (Huffman decode, range coder) and its host stages lie under the
    // issue-bound kernel A of another.  A large call is cut into that many chunks of about equal plane bytes; the
    // device memory budget `plane_cap` is shared by the chunks in flight.  Small calls stay in one piece.
    std::vector<std::pair<int, int>> ranges;
    int W = 1;
    {
        size_t total_need = 0;
        for (int i = 0; i < n; ++i) total_need += need[i];
        W = (n >= 64 && total_need >= (size_t(1) << 30)) ? std::max(1, c->concurrent) : 1;
        const size_t cap = c->plane_cap / (size_t)W;
        // LEPB200_CHUNK_SPLIT=s (tuning): s chunks per worker instead of one -- a shorter head (first kernel A) and tail (last
        // range coder + containers) against smaller launches of kernel A
        const int split = getenv("LEPB200_CHUNK_SPLIT") ? std::max(1, std::min(8, atoi(getenv("LEPB200_CHUNK_SPLIT")))) : 1;
        const size_t target = std::min(cap, std::max<size_t>(total_need / (size_t)(W * split) + 1, size_t(256) << 20));
        const int chunk = std::max(1, c->chunk_images);
        int b = 0;
        size_t acc = 0;
        for (int i = 0; i < n; ++i) {
            if (i > b && (i - b >= chunk || acc + need[i] > target)) { ranges.emplace_back(b, i); b = i; acc = 0; }
            acc += need[i];
        }
        ranges.emplace_back(b, n);
        if (c->chunk_images < 4096 && (int)ranges.size() > 1) W = std::max(W, std::min((int)ranges.size(), c->concurrent));   // caller-forced small chunks
        W = std::max(1, std::min(W, (int)ranges.size()));
    }
    keep_arenas_for(c, 1, W);
    const int pth = std::max(1, c->nthreads / W);          // host threads of one chunk's stages (W chunks share the cores)
    // Front stages take turns (LEPB200_FRONT_TURNS=0: all W at once, a W-th of the threads each): chunk 0's parse +
    // de-stuff + H2D with ALL host threads is done after a W-th of the time, so its Huffman kernels and kernel A start
    // while the other chunks are still being parsed, and the chunks reach the device one after the other instead of
    // all at the same moment (side by side, the fronts all end together and the chunks' Huffman launches then share the device).
    // containers assembled on the device (lepb200_encode_fetch_files) unless LEPB200_DEVICE_MUX=0 (host MuxWriter)
    const bool device_mux = !(getenv("LEPB200_DEVICE_MUX") && atoi(getenv("LEPB200_DEVICE_MUX")) == 0);
    const bool front_turns = W > 1 && !(getenv("LEPB200_FRONT_TURNS") && atoi(getenv("LEPB200_FRONT_TURNS")) == 0);
    const int fth = front_turns ? std::max(1, c->nthreads) : pth;
    std::mutex turn_mu;
    std::condition_variable turn_cv;
    int front_turn = 0;
    std::atomic<int> alive(W);                               // workers that still have a chunk to finish
    const int nchunks = (int)ranges.size();
    c->outputs.resize(n);
    std::vector<int> status(n, 0);
    std::vector<ChunkState> cs(nchunks);
    std::mutex tmu;

    auto front = [&](int k) {
        double t0 = now_s();
        ChunkState& s = cs[k];
        s.begin = ranges[k].first; s.end = ranges[k].second;
        const int m = s.end - s.begin;
        lepb200_ctx* ctx = c->ctx2[k % W];
        s.js.resize(m); s.planes.resize(m); s.splits.resize(m); s.host_decoded.assign(m, 0);
        // staging layout for the de-stuffed scans (a scan is never longer than its file) and arena layout for planes
        // of files that turn out to need the host decoder
        std::vector<size_t> soff(m + 1, 0), poff(m + 1, 0);
        for (int i = 0; i < m; ++i) {
            soff[i + 1] = soff[i] + ((jpegs[s.begin + i].len + 32 + 15) & ~size_t(15));
            poff[i + 1] = poff[i] + need[s.begin + i];
        }
        uint8_t* stage = c->gpu_huffman ? lepb200_huffman_stage_reserve(ctx, soff[m]) : nullptr;
        if (c->gpu_huffman && !stage) { s.gpu_rc = LEPB200_ERR_NOMEM; return; }
        const int slot = k % W;
        uint8_t* arena = nullptr;
        if (!c->gpu_huffman) {                       // every file takes the host decoder: one arena for the chunk
            if (!reserve_arena(c, slot, poff[m] + 256)) { s.gpu_rc = LEPB200_ERR_NOMEM; return; }
            arena = static_cast<uint8_t*>(c->arena[slot]);
        }
        std::vector<uint8_t> eligible(m, 0);
        std::vector<GpuScanSetup> setups(c->gpu_huffman ? m : 0);
        // pass 1: parse + de-stuff (into the staging buffer on the GPU path), in groups of consecutive files: a group's
        // staged bytes are contiguous, so one asynchronous H2D per group pushes them while other groups are still being
        // parsed (a copy per file would spend more time in the CUDA runtime than in the parser)
        const int group = 32, ngroups = (m + group - 1) / group;
        parallel_for(ngroups, fth, [&](int gi) {
            const int g0 = gi * group, g1 = std::min(m, g0 + group);
            for (int i = g0; i < g1; ++i) {
                s.js[i].reset(new Jpeg());
                Jpeg& j = *s.js[i];
                const lepb200_buffer& in = jpegs[s.begin + i];
                if (stage) { j.huff.attach(stage + soff[i], soff[i + 1] - soff[i] - 16); memset(stage + soff[i], 0, 16); }
                if (need[s.begin + i] > c->plane_cap / (size_t)W) { j.status = NOT_HANDLED; j.error = "image larger than the per-chunk device memory budget"; continue; }
                const bool parsed = parse_jpeg(in.data, in.len, j, c->embedding, c->discard_meta);
                if (stage) memset(stage + soff[i] + j.huff.size(), 0, 16);          // the decoder reads whole words past the end
                if (parsed && stage && gpu_scan_setup(j, setups[i])) eligible[i] = 1;
            }
            if (stage) lepb200_huffman_stage_upload(ctx, soff[g0], soff[g1] - soff[g0]);
        });
        // host-decoded files of a GPU chunk share one arena sized for just them
        if (c->gpu_huffman) {
            size_t tot = 0;
            std::vector<size_t> off(m, 0);
            for (int i = 0; i < m; ++i) if (!eligible[i] && s.js[i]->status == 0) { off[i] = tot; tot += need[s.begin + i]; }
            if (tot) {
                if (!reserve_arena(c, slot, tot + 256)) { s.gpu_rc = LEPB200_ERR_NOMEM; return; }
                arena = static_cast<uint8_t*>(c->arena[slot]);
            }
            for (int i = 0; i < m; ++i) poff[i] = off[i];
        }
        // pass 2: host Huffman decode where needed
        parallel_for(m, fth, [&](int i) {
            Jpeg& j = *s.js[i];
            for (int q = 0; q < 4; ++q) s.planes[i][q] = nullptr;
            if (j.status || eligible[i]) return;
            size_t want = 0;
            for (int q = 0; q < j.ncmp; ++q) want += (plane_bytes(j, q) + 255) & ~size_t(255);
            if (want != need[s.begin + i]) { j.status = NOT_HANDLED; j.error = "plane size peek mismatch"; return; }
            uint8_t* p = arena + poff[i];
            for (int q = 0; q < j.ncmp; ++q) {
                s.planes[i][q] = reinterpret_cast<int16_t*>(p);
                const size_t pb = plane_bytes(j, q);
                memset(p, 0, pb);
                p += (pb + 255) & ~size_t(255);
            }
            if (decode_scans(j, s.planes[i].data())) {
                // -rejectprogressive: the reference leaves with PROGRESSIVE_UNSUPPORTED at the first scan that is progressive
                // or does not interleave all components (jpgcoder.cc:2911-2925)
                if (!c->allow_progressive && !j.is_baseline) { j.status = PROGRESSIVE_UNSUPPORTED; j.error = "progressive / non-interleaved JPEG rejected (-rejectprogressive)"; return; }
                s.splits[i] = select_splits(j, c->max_encode_threads, c->min_encode_threads, c->even_split); s.host_decoded[i] = 1;
            }
        });
        // batch = every file that is still fine, in file order
        for (int i = 0; i < m; ++i) {
            status[s.begin + i] = s.js[i]->status;
            if (s.js[i]->status == 0) s.idx.push_back(i);
        }
        const int nb = (int)s.idx.size();
        s.scans.assign(nb, lepb200_jpeg_scan());
        s.rowbuf.resize(nb);
        for (int q = 0; q < nb; ++q) {
            const int i = s.idx[q];
            const Jpeg& j = *s.js[i];
            lepb200_jpeg_scan& sc = s.scans[q];
            fill_jpeg_scan(j, eligible[i] ? &setups[i] : nullptr, sc);
            if (!eligible[i]) continue;              // placeholder: plane slot only
            s.rowbuf[q].resize((size_t)j.mcuv + 1);
            sc.rows = s.rowbuf[q].data();
            s.any_gpu_huffman = true;
        }
        mark("front", k, t0);
        std::lock_guard<std::mutex> g(tmu);
        c->t_front += now_s() - t0;
    };

    auto gpu = [&](int k) {
        double t0 = now_s();
        ChunkState& s = cs[k];
        lepb200_ctx* ctx = c->ctx2[k % W];
        const int nb = (int)s.idx.size();
        if (s.gpu_rc == 0 && nb > 0) {
            if (s.any_gpu_huffman) {
                s.gpu_rc = lepb200_huffman_decode_to_device(ctx, s.scans.data(), nb);
                c->t_huff_ms = lepb200_last_huffman_ms(ctx);
                mark("huffman", k, t0);
                if (trace) fprintf(stderr, "[trace]   huffman kernels %.1f ms, %d synchronisation iterations, %d images redone by the serial kernel\n",
                                 c->t_huff_ms, lepb200_last_huffman_iterations(ctx), lepb200_last_huffman_redone(ctx));
            }
            double t1 = now_s();
            s.imgs.resize(nb);
            if (s.gpu_rc == 0) {
                // thread-segment selection from the Huffman states at the MCU-row starts (write_ujpg, jpgcoder.cc:3860-3934)
                parallel_for(nb, pth, [&](int q) {
                    const int i = s.idx[q];
                    Jpeg& j = *s.js[i];
                    const lepb200_jpeg_scan& sc = s.scans[q];
                    if (!s.host_decoded[i]) {
                        if (sc.status == 0 && sc.nrows >= 2) {
                            j.padbit = (int8_t)sc.padbit;
                            j.rows.clear();
                            for (int r = 0; r < sc.nrows; ++r) {
                                j.rows.push_back(handoff_from_state(j, sc.rows[r].bitpos, sc.rows[r].mcu_y, sc.rows[r].lastdc));
                                j.rows.back().tokens = sc.rows[r].tokens;
                            }
                            for (size_t r = 1; r < j.rows.size(); ++r)
                                if (j.rows[r].luma_y_start < j.rows[r - 1].luma_y_end) j.rows[r].luma_y_start = j.rows[r - 1].luma_y_end;
                            for (int t = 0; t < j.ncmp; ++t) { j.trunc_bcv[t] = j.cmp[t].bcv; j.trunc_bc[t] = j.cmp[t].bc; }
                            s.splits[i] = select_splits(j, c->max_encode_threads, c->min_encode_threads, c->even_split);
                        } else {
                            j.status = sc.status ? sc.status : (int)UNSUPPORTED_JPEG;
                            j.error = "GPU Huffman decoder refused the scan";
                            Handoff h0;                       // placeholder single segment so that the batch layout stays intact
                            s.splits[i].selected.assign(1, h0);
                        }
                        status[s.begin + i] = j.status;
                    }
                    fill_image(s.imgs[q], j, s.planes[i].data(), s.splits[i].selected);
                    if (!s.host_decoded[i] && j.status == 0) {
                        // decision-count bound of each thread-segment from the per-row counters of the Huffman kernel
                        lepb200_image& im = s.imgs[q];
                        size_t r = 0;
                        uint32_t start_tok[LEPB200_MAX_SEGMENTS + 1];
                        for (int t = 0; t < im.nseg; ++t) {
                            while (r + 1 < j.rows.size() && (int)j.rows[r].luma_y_start < im.luma_y_start[t]) ++r;
                            start_tok[t] = j.rows[r].tokens;
                        }
                        start_tok[im.nseg] = j.rows.back().tokens;
                        for (int t = 0; t < im.nseg; ++t) im.seg_token_bound[t] = std::max<uint32_t>(1u, start_tok[t + 1] - start_tok[t]);
                    }
                });
                int nseg_total = 0;
                s.seg_base.assign(nb + 1, 0);
                for (int q = 0; q < nb; ++q) { s.seg_base[q + 1] = s.seg_base[q] + s.imgs[q].nseg; nseg_total += s.imgs[q].nseg; }
                s.streams.resize(nseg_total);
                mark("segments", k, t1);
                t1 = now_s();
                s.gpu_rc = s.any_gpu_huffman ? lepb200_encode_upload_resident(ctx, s.imgs.data(), nb) : lepb200_encode_upload(ctx, s.imgs.data(), nb);
                mark("upload+prepass", k, t1);
                t1 = now_s();
                if (s.gpu_rc == 0) s.gpu_rc = lepb200_encode_launch(ctx);
                if (device_mux) {
                    // while the kernels run: the part of every container that does not depend on the coded bytes (fixed
                    // header, zlib'd JPEG header, "CMP"); then the files themselves come back assembled by the device
                    s.headers.assign(nb, std::vector<uint8_t>());
                    std::vector<lepb200_buffer> hb(nb, lepb200_buffer{nullptr, 0});
                    parallel_for(nb, pth, [&](int q) {
                        const int i = s.idx[q];
                        if (status[s.begin + i]) return;
                        std::string err;
                        if (build_lep_header(*s.js[i], s.splits[i], s.headers[q], err)) hb[q] = lepb200_buffer{s.headers[q].data(), s.headers[q].size()};
                    });
                    s.files.assign(nb, lepb200_result{nullptr, 0, 0});
                    if (s.gpu_rc == 0) s.gpu_rc = lepb200_encode_fetch_files(ctx, hb.data(), s.files.data());
                } else if (s.gpu_rc == 0) s.gpu_rc = lepb200_encode_fetch(ctx, s.streams.data());
                mark("encode+fetch", k, t1);
                if (trace) fprintf(stderr, "[trace]   kernel A %.1f ms, A+B %.1f ms\n", lepb200_last_symbolise_ms(ctx), lepb200_last_kernel_ms(ctx));
            }
        }
        std::lock_guard<std::mutex> g(tmu);
        c->t_gpu += now_s() - t0;
    };

    auto back = [&](int k) {
        double t0 = now_s();
        ChunkState& s = cs[k];
        // the workers that have no chunk left leave their share of the host threads to the ones still writing containers
        const int bth = std::max(pth, c->nthreads / std::max(1, alive.load()));
        if (s.gpu_rc == 0) {
            parallel_for((int)s.idx.size(), bth, [&](int q) {
                const int i = s.begin + s.idx[q];
                if (status[i]) return;
                if (device_mux) {                     // the file is complete: it only moves into the codec's output buffer
                    const lepb200_result& f = s.files[q];
                    if (f.status) { status[i] = f.status; return; }
                    c->outputs[i].assign(f.data, f.data + f.len);
                    return;
                }
                std::vector<std::pair<const uint8_t*, size_t>> ss;
                for (int t = s.seg_base[q]; t < s.seg_base[q + 1]; ++t) {
                    if (s.streams[t].status) { status[i] = s.streams[t].status; return; }
                    ss.emplace_back(s.streams[t].data, (size_t)s.streams[t].len);
                }
                std::string err;
                c->outputs[i].clear();
                if (!write_lep(*s.js[s.idx[q]], s.splits[s.idx[q]], ss, c->outputs[i], err)) { status[i] = NOT_HANDLED; c->outputs[i].clear(); }
            });
        }
        parallel_for((int)s.js.size(), bth, [&](int i) { s.js[i].reset(); });     // release per-chunk host state early
        s.js.clear(); s.planes.clear(); s.splits.clear();
        mark("back", k, t0);
        std::lock_guard<std::mutex> g(tmu);
        c->t_back += now_s() - t0;
    };

    // W workers; worker w takes the chunks w, w + W, ... through front -> gpu -> back on context w.  Chunks of different
    // workers overlap freely: host stages with device stages, and on the device the kernels of different streams
    {
        std::vector<std::thread> workers;
        for (int w = 0; w < W; ++w)
            workers.emplace_back([&, w]() {
                for (int k = w; k < nchunks; k += W) {
                    if (front_turns) {
                        std::unique_lock<std::mutex> lk(turn_mu);
                        turn_cv.wait(lk, [&] { return front_turn == k; });
                    }
                    front(k);
                    if (front_turns) {
                        { std::lock_guard<std::mutex> lk(turn_mu); ++front_turn; }
                        turn_cv.notify_all();
                    }
                    gpu(k);
                    if (k + W >= nchunks) --alive;           // this worker's last chunk: only its container stage is left
                    back(k);
                }
            });
        for (auto& t : workers) t.join();
    }
    int ret = LEPB200_OK;
    for (int k = 0; k < nchunks; ++k)
        if (cs[k].gpu_rc) {               // the chunk's device work failed (e.g. out of memory): none of its files has an output
            ret = cs[k].gpu_rc; c->err = lepb200_last_error(c->ctx2[k % W]);
            for (int i = ranges[k].first; i < ranges[k].second; ++i) if (!status[i]) status[i] = 33;       // ExitCode::OS_ERROR
        }
    // -verify / -roundtrip (the reference CLI's default, jpgcoder.cc:1095-1110, validation.cc): every .lep is decoded
    // again and must give back the input byte for byte; a file that does not is withheld with ROUNDTRIP_FAILURE (41)
    if (c->verify && ret == LEPB200_OK) {
        std::vector<std::vector<uint8_t>> leps;
        leps.swap(c->outputs);
        std::vector<int> idx;
        std::vector<lepb200_buffer> vin;
        for (int i = 0; i < n; ++i) if (!status[i]) { idx.push_back(i); vin.push_back({leps[i].data(), leps[i].size()}); }
        if (!idx.empty()) {
            const double tf = c->t_front, tg = c->t_gpu, tb = c->t_back;
            std::vector<lepb200_result> back(idx.size(), lepb200_result{nullptr, 0, 0});
            const bool zlib0 = c->zlib0;                                         // the check compares plain JPEG bytes
            c->zlib0 = false;
            const int vrc = lepb200_decompress_leps(c, vin.data(), (int)vin.size(), back.data());
            c->zlib0 = zlib0;
            for (size_t q = 0; q < idx.size(); ++q) {
                const lepb200_buffer& src = jpegs[idx[q]];
                const bool same = vrc == LEPB200_OK && back[q].status == 0 && back[q].len == src.len && !memcmp(back[q].data, src.data, src.len);
                if (!same) status[idx[q]] = 41;                                    // ExitCode::ROUNDTRIP_FAILURE
            }
            c->t_front += tf; c->t_gpu += tg; c->t_back += tb;                   // the verification pass is part of the call
        }
        c->outputs.swap(leps);
    }
    for (int i = 0; i < n; ++i) {
        if (status[i]) c->outputs[i].clear();
        out[i].status = status[i];
        out[i].data = status[i] ? nullptr : c->outputs[i].data();
        out[i].len = status[i] ? 0 : c->outputs[i].size();
    }
    return ret;
}

// The job the device Huffman encoder gets for one .lep file (lepb200_huffman_encode_resident): tables selected by the SOS,
// sampling factors, and per thread-segment the MCU-row range, DC predictors, pending bits and byte count its ThreadHandoff
// carries (recode_row_range, src/lepton/recoder.cc:472-545).  he.scan_bytes stays 0 when the file needs the host re-encoder.
static void fill_henc_image(const LepFile& lf, GpuRecodeSetup& gs, lepb200_henc_image& he) {
    memset(&he, 0, sizeof(he));
    if (!gpu_recode_setup(lf, gs)) return;
    const Jpeg& j = lf.j;
    he.rsti = gs.rsti; he.padbit = (uint8_t)j.padbit;
    for (int t = 0; t < j.ncmp; ++t) {
        he.H[t] = j.cmp[t].H; he.V[t] = j.cmp[t].V;
        he.dc[t] = gs.dc[t]; he.ac[t] = gs.ac[t];
    }
    const int luma_mul = j.cmp[0].bcv / j.mcuv;
    he.nseg = lf.nseg;
    bool ok = lf.nseg >= 1 && lf.nseg <= LEPB200_MAX_SEGMENTS;
    for (int t = 0; ok && t < lf.nseg; ++t) {
        const Handoff& hd = lf.handoffs[t];
        lepb200_henc_segment& sg = he.seg[t];
        ok = hd.luma_y_start % luma_mul == 0 && hd.num_overhang_bits < 8;
        sg.mcu_row_start = hd.luma_y_start / luma_mul;
        sg.mcu_row_end = t + 1 < lf.nseg ? lf.handoffs[t + 1].luma_y_start / luma_mul : j.mcuv;
        for (int q3 = 0; q3 < 3; ++q3) sg.last_dc[q3] = hd.last_dc[q3];
        sg.overhang_bits = hd.num_overhang_bits; sg.overhang_byte = hd.overhang_byte;
        sg.expect_bytes = hd.segment_size;
    }
    if (ok) he.scan_bytes = gs.scan_bytes;
}

// .lep files -> JPEG files (inverse of lepb200_compress_jpegs), same 3-stage chunk pipeline:
//   front (host: container parse, zlib inflate, demux)  |  gpu (H2D streams, decode kernel, D2H planes)  |
//   back (host: Huffman re-encode + byte stuffing + header/garbage re-assembly)
int lepb200_decompress_leps(lepb200_codec* c, const lepb200_buffer* leps, int n, lepb200_result* out) {
    if (!c || !leps || !out || n <= 0) return LEPB200_ERR_INVALID;
    const bool trace = getenv("LEPB200_TRACE") != nullptr;           // stage timeline on stderr (diagnostics)
    const double t_origin = now_s();
    auto mark = [&](const char* what, int k, double t_begin) {
        if (trace) fprintf(stderr, "[trace] %-16s chunk %d  %8.1f -> %8.1f ms\n", what, k, (t_begin - t_origin) * 1e3, (now_s() - t_origin) * 1e3);
    };
    c->err.clear();
    c->t_front = c->t_gpu = c->t_back = 0;
    c->n_gpu_recoded = 0;
    // ---- containers: fixed header, zlib'd JPEG header, handoffs, demux of the segment streams (all files, host threads).
    // Every input may be a stream of concatenated .lep files: each of its members is one image of the batch below, so the
    // members of one input and those of different inputs share chunks, kernels and host stages alike.
    double t_parse = now_s();
    std::vector<std::vector<std::unique_ptr<LepFile>>> members(n);
    parallel_for(n, c->nthreads, [&](int i) { read_lep_members(leps[i].data, leps[i].len, members[i], /*lazy=*/true); });   // mux packets stay where they are: gathered into the staging buffer
    std::vector<int> first(n + 1, 0);                 // members of input i: images first[i] .. first[i + 1] - 1
    for (int i = 0; i < n; ++i) first[i + 1] = first[i] + (int)members[i].size();
    const int nim = first[n];
    std::vector<std::unique_ptr<LepFile>> all(nim);
    std::vector<uint8_t> zjoin(nim, 0);               // 1: a member of an input of several members that goes out as one zlib stream
    for (int i = 0; i < n; ++i) {
        const bool z = members[i].size() > 1 && (c->zlib0 || members[i][0]->zlib0);
        for (size_t m = 0; m < members[i].size(); ++m) { zjoin[first[i] + m] = z; all[first[i] + m] = std::move(members[i][m]); }
    }
    std::vector<size_t> pbytes(nim, 0);
    parallel_for(nim, c->nthreads, [&](int u) {
        if (all[u]->status) return;
        for (int q = 0; q < all[u]->j.ncmp; ++q) pbytes[u] += (plane_bytes(all[u]->j, q) + 255) & ~size_t(255);
        if (pbytes[u] > c->plane_cap) { all[u]->status = NOT_HANDLED; all[u]->error = "image larger than the per-chunk device memory budget"; pbytes[u] = 0; }
    });
    std::vector<uint32_t> member_adler(nim, 1);       // zjoin images: Adler-32 of the restored member
    c->t_front += now_s() - t_parse;
    mark("containers", -1, t_parse);
    // chunks of up to `plane_cap` bytes of coefficient planes (device memory: three contexts in flight).  The planes stay on the device
    // for every file whose scan the GPU can re-encode; only the others need a pinned host arena (128 B per block over PCIe)
    std::vector<std::pair<int, int>> ranges;
    int W = 1;
    {
        // Unlike the way in, the way back wants LARGE chunks: the decode kernel of large batches (lep_decode_g2.cu, eight
        // serial chains per warp) is bound by the latency of a chain, so its duration hardly depends on how many
        // segments a launch covers -- cutting a call into four chunks costs four times that latency.  A chunk therefore takes as much as the device memory budget
        // allows; when a call needs several, two are in flight (the second one's host stages and copies under the
        // first one's kernel).  Without the device re-encoder every plane needs pinned host memory too: small chunks.
        // The two chunks in flight share the budget when a call does not fit in one.
        const size_t budget = c->gpu_huffman ? c->plane_cap : (size_t(6) << 30);
        size_t total = 0;
        for (int i = 0; i < nim; ++i) total += pbytes[i];
        const size_t cap = total > budget ? budget / 2 : budget;
        const int chunk_max = std::max(1, c->chunk_images);
        int b0 = 0;
        size_t acc = 0;
        for (int i = 0; i < nim; ++i) {
            if (i > b0 && (i - b0 >= chunk_max || acc + pbytes[i] > cap)) { ranges.emplace_back(b0, i); b0 = i; acc = 0; }
            acc += pbytes[i];
        }
        ranges.emplace_back(b0, nim);
        W = std::max(1, std::min(std::min(2, c->concurrent), (int)ranges.size()));
    }
    keep_arenas_for(c, 2, W);
    const int pth = std::max(1, c->nthreads / W);
    const int nchunks = (int)ranges.size();
    // the output buffers keep their capacity from call to call (a fresh 1.5 GB of vectors per 4096-file call is 370 K
    // page faults inside the container stage); every image's buffer is rewritten or cleared below.  Indices from here on
    // are images (members), not inputs.
    c->outputs.resize(nim);
    for (auto& o : c->outputs) o.clear();
    std::vector<int> status(nim, 0);
    struct DChunk {
        int begin = 0, end = 0;
        std::vector<std::unique_ptr<LepFile>> lf;
        std::vector<std::array<int16_t*, 4>> planes;        // host planes of the files the host re-encodes (else null)
        std::vector<lepb200_image> imgs;
        std::vector<int> idx;
        std::vector<lepb200_stream> streams;
        std::vector<lepb200_buffer> spans;          // mux packets of all streams of the chunk, in stream order
        std::vector<uint32_t> span_first;           // per stream: its first packet in `spans` (+ one past the end)
        std::vector<int32_t> seg_status;
        std::vector<int> seg_base;
        std::vector<lepb200_henc_image> henc;       // per batch image: scan re-encoded on the device when scan_bytes != 0
        std::vector<GpuRecodeSetup> gsetup;
        std::vector<std::vector<int16_t>> fallback;  // planes of files whose device re-encode did not check out
        int gpu_rc = 0;
    };
    std::vector<DChunk> cs(nchunks);
    std::mutex tmu;
    auto front = [&](int k) {
        double t0 = now_s();
        DChunk& s = cs[k];
        s.begin = ranges[k].first; s.end = ranges[k].second;
        const int m = s.end - s.begin;
        s.lf.resize(m); s.planes.resize(m);
        for (int i = 0; i < m; ++i) {
            s.lf[i] = std::move(all[s.begin + i]);
            status[s.begin + i] = s.lf[i]->status;
            for (int q = 0; q < 4; ++q) s.planes[i][q] = nullptr;
            if (s.lf[i]->status == 0) s.idx.push_back(i);
        }
        const int nb = (int)s.idx.size();
        // GPU Huffman re-encode set-up for the files that allow it (complete single-scan baseline)
        s.henc.assign(nb, lepb200_henc_image());
        s.gsetup.assign(nb, GpuRecodeSetup());
        s.fallback.resize(nb);
        parallel_for(nb, pth, [&](int q) {
            const LepFile& lf = *s.lf[s.idx[q]];
            lepb200_henc_image& he = s.henc[q];
            memset(&he, 0, sizeof(he));
            if (c->gpu_huffman) fill_henc_image(lf, s.gsetup[q], he);
        });
        // pinned arena for the planes of the files the host re-encodes
        size_t total = 0;
        std::vector<size_t> base(nb, 0);
        for (int q = 0; q < nb; ++q) if (s.henc[q].scan_bytes == 0) { base[q] = total; total += pbytes[s.begin + s.idx[q]]; }
        uint8_t* arena = nullptr;
        if (total) {
            if (!reserve_arena(c, k % W, total + 256)) { s.gpu_rc = LEPB200_ERR_NOMEM; return; }
            arena = static_cast<uint8_t*>(c->arena[k % W]);
        }
        int nseg_total = 0;
        s.imgs.resize(nb);
        for (int q = 0; q < nb; ++q) {
            const int i = s.idx[q];
            LepFile& lf = *s.lf[i];
            const Jpeg& j = lf.j;
            if (s.henc[q].scan_bytes == 0) {
                uint8_t* p = arena + base[q];
                for (int t = 0; t < j.ncmp; ++t) { s.planes[i][t] = reinterpret_cast<int16_t*>(p); p += (plane_bytes(j, t) + 255) & ~size_t(255); }
            }
            fill_image(s.imgs[q], j, s.planes[i].data(), lf.handoffs);
            // files that stay on the device have no host planes; the batch builder only wants the pointers non-null
            for (int t = 0; t < j.ncmp; ++t) if (!s.imgs[q].planes[t]) s.imgs[q].planes[t] = reinterpret_cast<int16_t*>(uintptr_t(1));
            for (int t = 0; t < lf.nseg; ++t) {
                lepb200_stream st;
                memset(&st, 0, sizeof(st));
                st.data = nullptr;
                st.len = lf.stream_len[t];
                s.span_first.push_back((uint32_t)s.spans.size());
                for (const auto& sp : lf.spans[t]) s.spans.push_back(lepb200_buffer{sp.first, sp.second});
                s.streams.push_back(st);
            }
            nseg_total += lf.nseg;
        }
        s.span_first.push_back((uint32_t)s.spans.size());
        s.seg_status.assign(nseg_total, 0);
        s.seg_base.assign(nb + 1, 0);
        for (int q = 0; q < nb; ++q) s.seg_base[q + 1] = s.seg_base[q] + s.imgs[q].nseg;
        mark("front", k, t0);
        std::lock_guard<std::mutex> g(tmu);
        c->t_front += now_s() - t0;
    };
    // parts of the device Huffman encode whose D2H and JPEG assembly run under the encode of the next part
    // (LEPB200_HENC_PARTS, 1 = one launch, everything after it as before round 2's last change)
    const int henc_parts_want = getenv("LEPB200_HENC_PARTS") ? std::max(1, std::min(16, atoi(getenv("LEPB200_HENC_PARTS")))) : 4;
    // zlib0 output (codec setting, or a zeta-headed file): the Adler-32 of a device-encoded scan comes from the encode kernel
    // unless LEPB200_ZLIB0_HOST_ADLER=1, which has the host sum every byte (the route of host-encoded files) for comparison
    const bool zlib0_host_adler = getenv("LEPB200_ZLIB0_HOST_ADLER") && atoi(getenv("LEPB200_ZLIB0_HOST_ADLER")) != 0;
    auto out_mode = [&](const LepFile& lf, bool device_scan) {
        if (!c->zlib0 && !lf.zlib0) return JpegOut::plain;       // a member's magic is its stream's first member's
        return device_scan && !zlib0_host_adler ? JpegOut::zlib0_scan_adler : JpegOut::zlib0_host_adler;
    };
    auto gpu = [&](int k) {               // H2D of the streams + decode kernel + Huffman encode of the resident planes, all queued
        double t0 = now_s();
        DChunk& s = cs[k];
        lepb200_ctx* ctx = c->ctx2[k % W];
        if (s.gpu_rc == 0 && !s.imgs.empty()) {
            s.gpu_rc = lepb200_decode_upload_gather(ctx, s.imgs.data(), (int)s.imgs.size(), s.streams.data(), s.spans.data(), s.span_first.data());
            mark("pack+upload", k, t0);
            if (s.gpu_rc == 0) s.gpu_rc = lepb200_decode_launch(ctx);
            const int parts = s.imgs.size() >= 256 ? henc_parts_want : 1;
            if (s.gpu_rc == 0) s.gpu_rc = lepb200_huffman_encode_resident_parts(ctx, s.henc.data(), (int)s.henc.size(), parts);   // scans re-encoded from the resident planes
        }
        std::lock_guard<std::mutex> g(tmu);
        c->t_gpu += now_s() - t0;
    };
    // JPEG of one batch image from the scan the device produced
    auto assemble = [&](DChunk& s, int q, uint32_t scan_adler) {
        const int li = s.idx[q], i = s.begin + li;
        for (int t = s.seg_base[q]; t < s.seg_base[q + 1]; ++t)
            if (s.seg_status[t]) { status[i] = s.seg_status[t]; return; }
        std::string err;
        c->n_gpu_recoded++;
        const LepFile& lf = *s.lf[li];
        if (!assemble_baseline(lf, s.gsetup[q], s.henc[q].data, c->outputs[i], err, out_mode(lf, true), scan_adler, zjoin[i] ? &member_adler[i] : nullptr)) { status[i] = NOT_HANDLED; c->outputs[i].clear(); }
    };
    auto fetch_back = [&](int k) {
        double t0 = now_s();
        DChunk& s = cs[k];
        const int nb = (int)s.imgs.size();
        std::vector<uint8_t> done(nb, 0);
        std::vector<uint32_t> scan_adler(nb, 1);
        bool kernel_adler = false;                      // some file of the chunk takes its scan's Adler-32 from the encode kernel
        for (int q = 0; q < nb; ++q) kernel_adler |= out_mode(*s.lf[s.idx[q]], true) == JpegOut::zlib0_scan_adler;
        lepb200_ctx* ctx = nb ? c->ctx2[k % W] : nullptr;
        if (s.gpu_rc == 0 && nb) {
            // decode status as soon as the decode kernel is through, then the parts of the device re-encode as they arrive
            s.gpu_rc = lepb200_decode_fetch_status(ctx, s.seg_status.data());
            mark("decode", k, t0);
            const int parts = s.gpu_rc == 0 ? lepb200_huffman_encode_parts(ctx) : 0;
            for (int p = 0; p < parts && s.gpu_rc == 0; ++p) {
                double tp = now_s();
                int q0 = 0, q1 = 0;
                s.gpu_rc = lepb200_huffman_encode_wait_part(ctx, s.henc.data(), nb, p, &q0, &q1);
                if (s.gpu_rc == 0 && kernel_adler) s.gpu_rc = lepb200_huffman_encode_adler32(ctx, q0, q1, scan_adler.data());
                if (s.gpu_rc) break;
                mark("huffenc part", k, tp);
                tp = now_s();
                parallel_for(q1 - q0, pth, [&](int d) {
                    const int q = q0 + d;
                    const lepb200_henc_image& he = s.henc[q];
                    if (!(he.scan_bytes && he.status == 0 && he.data)) return;
                    assemble(s, q, scan_adler[q]);
                    done[q] = 1;
                });
                mark("assemble part", k, tp);
            }
        }
        double t1 = now_s();
        if (s.gpu_rc == 0 && nb) {
            // planes come back only for the files the host has to re-encode
            std::vector<lepb200_image> need(s.imgs);
            for (int q = 0; q < nb; ++q) {
                const lepb200_henc_image& he = s.henc[q];
                const int li = s.idx[q];
                const Jpeg& j = s.lf[li]->j;
                if (done[q]) { for (int t = 0; t < 3; ++t) need[q].planes[t] = nullptr; continue; }
                if (he.scan_bytes == 0) continue;                                  // planned for the host: arena pointers are in place
                // the device re-encode did not produce the byte counts the handoffs promise: fetch the planes after all
                size_t tot = 0;
                for (int t = 0; t < j.ncmp; ++t) tot += plane_bytes(j, t) / 2;
                s.fallback[q].assign(tot, 0);
                int16_t* p = s.fallback[q].data();
                for (int t = 0; t < j.ncmp; ++t) { s.planes[li][t] = p; need[q].planes[t] = p; p += plane_bytes(j, t) / 2; }
            }
            s.gpu_rc = lepb200_decode_fetch(ctx, need.data(), nb, s.seg_status.data());
            if (trace) fprintf(stderr, "[trace]   decode kernel %.1f ms\n", lepb200_last_kernel_ms(ctx));
        }
        mark("fetch", k, t1);
        t1 = now_s();
        if (s.gpu_rc == 0) {
            parallel_for(nb, pth, [&](int q) {
                if (done[q]) return;
                const int li = s.idx[q], i = s.begin + li;
                for (int t = s.seg_base[q]; t < s.seg_base[q + 1]; ++t)
                    if (s.seg_status[t]) { status[i] = s.seg_status[t]; return; }
                std::string err;
                const LepFile& lf = *s.lf[li];
                if (!recode_baseline(lf, s.planes[li].data(), c->outputs[i], err, out_mode(lf, false), zjoin[i] ? &member_adler[i] : nullptr)) { status[i] = NOT_HANDLED; c->outputs[i].clear(); }
            });
        }
        s.lf.clear();
        mark("back", k, t1);
        std::lock_guard<std::mutex> g(tmu);
        c->t_gpu += t1 - t0;
        c->t_back += now_s() - t1;
    };
    // W workers; worker w takes the chunks w, w + W, ... through front -> gpu -> fetch -> back on context / arena w
    {
        std::vector<std::thread> workers;
        for (int w = 0; w < W; ++w)
            workers.emplace_back([&, w]() {
                for (int k = w; k < nchunks; k += W) { front(k); gpu(k); fetch_back(k); }
            });
        for (auto& t : workers) t.join();
    }
    int rc = LEPB200_OK;
    for (int k = 0; k < nchunks; ++k)
        if (cs[k].gpu_rc) {
            rc = cs[k].gpu_rc; c->err = lepb200_last_error(c->ctx2[k % W]);
            for (int i = ranges[k].first; i < ranges[k].second; ++i) if (!status[i]) status[i] = 33;       // ExitCode::OS_ERROR
        }
    // back to inputs: the status of the first member that failed, else the members' JPEGs one after the other (one zlib
    // stream over all of them for zlib0 output).  A single member's buffer is handed out as it is.
    c->joined.resize(n);
    parallel_for(n, c->nthreads, [&](int i) {
        int st = 0;
        for (int u = first[i]; u < first[i + 1] && !st; ++u) st = status[u];
        std::vector<uint8_t>* o = &c->outputs[first[i]];
        if (!st && first[i + 1] - first[i] > 1) {
            std::vector<std::pair<const uint8_t*, size_t>> parts;
            for (int u = first[i]; u < first[i + 1]; ++u) parts.emplace_back(c->outputs[u].data(), c->outputs[u].size());
            o = &c->joined[i];
            o->clear();
            if (zjoin[first[i]]) zlib0_join(parts, &member_adler[first[i]], *o);
            else for (const auto& pc : parts) o->insert(o->end(), pc.first, pc.first + pc.second);
        }
        out[i].status = st;
        out[i].data = st ? nullptr : o->data();
        out[i].len = st ? 0 : o->size();
    });
    return rc;
}

// ---- host-only decode-side stages (no GPU): parse a .lep, expose geometry/streams, re-create the JPEG from planes
struct lepb200_lep {
    LepFile lf;
    std::vector<uint8_t> out;
};
int lepb200_host_lep_open(const uint8_t* data, size_t len, lepb200_lep** out, int32_t* status) {
    if (!out || !data) return LEPB200_ERR_INVALID;
    lepb200_lep* h = new lepb200_lep();
    *out = h;
    read_lep(data, len, h->lf);
    if (status) *status = h->lf.status;
    return LEPB200_OK;
}
const char* lepb200_host_lep_error(const lepb200_lep* h) { return h ? h->lf.error.c_str() : "null"; }
// geometry + splits (planes pointers are left null: the caller provides the planes)
int lepb200_host_lep_image(lepb200_lep* h, lepb200_image* img) {
    if (!h || !img || h->lf.status) return LEPB200_ERR_INVALID;
    int16_t* none[4] = {nullptr, nullptr, nullptr, nullptr};
    fill_image(*img, h->lf.j, none, h->lf.handoffs);
    return LEPB200_OK;
}
int lepb200_host_lep_stream(lepb200_lep* h, int seg, const uint8_t** data, size_t* len) {
    if (!h || h->lf.status || seg < 0 || seg >= h->lf.nseg) return LEPB200_ERR_INVALID;
    *data = h->lf.streams[seg].data();
    *len = h->lf.streams[seg].size();
    return LEPB200_OK;
}
int lepb200_host_lep_recode(lepb200_lep* h, const int16_t* const planes[3], const uint8_t** data, size_t* len) {
    if (!h || h->lf.status) return LEPB200_ERR_INVALID;
    const int16_t* p4[4] = {planes[0], planes[1], planes[2], nullptr};
    std::string err;
    if (!recode_baseline(h->lf, p4, h->out, err)) { h->lf.error = err; return LEPB200_ERR_INVALID; }
    *data = h->out.data();
    *len = h->out.size();
    return LEPB200_OK;
}
// Host half of the device re-encode path: where the scan lies in the original file (0 = the file needs the host
// re-encoder) and the assembly of the JPEG around scan bytes produced elsewhere.
int lepb200_host_lep_scan_layout(lepb200_lep* h, uint32_t* scan_offset, uint32_t* scan_bytes) {
    if (!h || h->lf.status || !scan_offset || !scan_bytes) return LEPB200_ERR_INVALID;
    GpuRecodeSetup gs;
    if (!gpu_recode_setup(h->lf, gs)) { *scan_offset = 0; *scan_bytes = 0; return LEPB200_OK; }
    *scan_offset = (uint32_t)(h->lf.j.prefix.size() + 2 + gs.hpos);
    *scan_bytes = gs.scan_bytes;
    return LEPB200_OK;
}
// Test hook (host only): the container parsed both ways -- streams copied out, and mux packets recorded in place (what
// lepb200_decompress_leps hands to lepb200_decode_upload_gather) -- must agree on status, segment count and every stream byte.
int lepb200_host_lep_lazy_equal(const uint8_t* data, size_t len) {
    if (!data) return LEPB200_ERR_INVALID;
    LepFile a, b;
    const bool ra = read_lep(data, len, a, false), rb = read_lep(data, len, b, true);
    if (ra != rb || a.status != b.status) return 1;
    if (!ra) return 0;
    if (a.nseg != b.nseg || (int)a.streams.size() != a.nseg || (int)b.spans.size() != b.nseg || !b.streams.empty()) return 2;
    for (int t = 0; t < a.nseg; ++t) {
        if (a.streams[t].size() != b.stream_len[t]) return 3;
        size_t off = 0;
        for (const auto& sp : b.spans[t]) {
            if (off + sp.second > a.streams[t].size() || memcmp(a.streams[t].data() + off, sp.first, sp.second)) return 4;
            off += sp.second;
        }
        if (off != a.streams[t].size()) return 5;
    }
    return 0;
}
int lepb200_host_brotli_available(void) { return brotli_available() ? 1 : 0; }
int lepb200_host_lep_members(const uint8_t* data, size_t len, lepb200_lep_member* out, int cap) {
    if (!data || (cap > 0 && !out)) return LEPB200_ERR_INVALID;
    std::vector<std::unique_ptr<LepFile>> ms;
    read_lep_members(data, len, ms, /*lazy=*/true);
    for (size_t k = 0; k < ms.size() && (int)k < cap; ++k) out[k] = lepb200_lep_member{ms[k]->status, ms[k]->jpeg_size, ms[k]->nseg};
    return (int)ms.size();
}
int lepb200_host_lep_open_member(const uint8_t* data, size_t len, int index, lepb200_lep** out, int32_t* status) {
    if (!out || !data) return LEPB200_ERR_INVALID;
    std::vector<std::unique_ptr<LepFile>> ms;
    read_lep_members(data, len, ms, /*lazy=*/false);
    if (index < 0 || index >= (int)ms.size()) return LEPB200_ERR_INVALID;
    lepb200_lep* h = new lepb200_lep();
    h->lf = std::move(*ms[index]);
    *out = h;
    if (status) *status = h->lf.status;
    return LEPB200_OK;
}
int lepb200_host_lep_henc_image(lepb200_lep* h, lepb200_henc_image* out) {
    if (!h || h->lf.status || !out) return LEPB200_ERR_INVALID;
    GpuRecodeSetup gs;
    fill_henc_image(h->lf, gs, *out);
    return LEPB200_OK;
}
int lepb200_host_lep_assemble(lepb200_lep* h, const uint8_t* scan, size_t scan_len, const uint8_t** data, size_t* len) {
    if (!h || h->lf.status || !scan) return LEPB200_ERR_INVALID;
    GpuRecodeSetup gs;
    if (!gpu_recode_setup(h->lf, gs) || gs.scan_bytes != scan_len) return LEPB200_ERR_INVALID;
    std::string err;
    if (!assemble_baseline(h->lf, gs, scan, h->out, err)) { h->lf.error = err; return LEPB200_ERR_INVALID; }
    *data = h->out.data();
    *len = h->out.size();
    return LEPB200_OK;
}
void lepb200_host_lep_close(lepb200_lep* h) { delete h; }
int lepb200_host_lep_zlib0(const lepb200_lep* h) { return h && h->lf.zlib0 ? 1 : 0; }
size_t lepb200_host_zlib0_frame(const uint8_t* data, size_t len, uint8_t* out, size_t cap) {
    if (!data && len) return 0;
    const size_t need = zlib0_size(len);
    if (out && cap >= need) {
        std::vector<uint8_t> framed;
        zlib0_frame(data, len, framed);
        memcpy(out, framed.data(), need);
    }
    return need;
}

// Host front end only (parse + Huffman decode + split selection) over a batch with `threads` workers; returns the
// wall-clock seconds.  Diagnostic: lets the host stage be profiled without a GPU.
double lepb200_host_frontend_seconds(const lepb200_buffer* jpegs, int n, int threads, int32_t* first_error) {
    std::vector<std::unique_ptr<Jpeg>> js(n);
    std::vector<std::vector<int16_t>> store(n);
    double t0 = now_s();
    parallel_for(n, threads, [&](int i) {
        js[i].reset(new Jpeg());
        Jpeg& j = *js[i];
        if (!parse_jpeg(jpegs[i].data, jpegs[i].len, j)) return;
        size_t total = 0;
        for (int k = 0; k < j.ncmp; ++k) total += (size_t)j.cmp[k].bc * 64;
        store[i].assign(total, 0);
        int16_t* planes[4] = {nullptr, nullptr, nullptr, nullptr};
        size_t off = 0;
        for (int k = 0; k < j.ncmp; ++k) { planes[k] = store[i].data() + off; off += (size_t)j.cmp[k].bc * 64; }
        if (decode_scans(j, planes)) select_splits(j);
    });
    double dt = now_s() - t0;
    if (first_error) { *first_error = 0; for (int i = 0; i < n; ++i) if (js[i]->status) { *first_error = js[i]->status; break; } }
    return dt;
}

// ---- several GPUs from one process (SURVEY 8(e): per-GPU work queues, no collective, no peer traffic) ----------------
// Files are independent, so the batch is dealt to the codecs (one per GPU) longest-first by size -- every GPU gets
// the same number of bytes to within one file -- and every codec runs its share through its own chunk pipeline on its
// own host thread.  A chunk has to stay large (the Huffman and range-coder kernels are latency-bound chains whose
// duration hardly depends on the number of files), which is why the split is static per call and not file by file.
void lepb200_shard_by_size(const size_t* sizes, int n, int world, int* owner) {
    if (!sizes || !owner || n <= 0 || world <= 0) return;
    std::vector<int> order(n);
    for (int i = 0; i < n; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return sizes[a] > sizes[b]; });
    std::vector<unsigned long long> load(world, 0);
    for (int i : order) {
        int r = 0;
        for (int k = 1; k < world; ++k) if (load[k] < load[r]) r = k;
        owner[i] = r;
        load[r] += sizes[i];
    }
}

namespace {
int run_multi(lepb200_codec* const* codecs, int ncodecs, const lepb200_buffer* in, int n, lepb200_result* out, bool compress) {
    if (!codecs || ncodecs <= 0 || !in || !out || n <= 0) return LEPB200_ERR_INVALID;
    for (int k = 0; k < ncodecs; ++k) if (!codecs[k]) return LEPB200_ERR_INVALID;
    std::vector<size_t> sizes(n);
    for (int i = 0; i < n; ++i) sizes[i] = in[i].len;
    std::vector<int> owner(n, 0);
    lepb200_shard_by_size(sizes.data(), n, ncodecs, owner.data());
    std::vector<std::vector<int>> share(ncodecs);
    for (int i = 0; i < n; ++i) share[owner[i]].push_back(i);                       // file order inside a share
    std::vector<int> rcs(ncodecs, LEPB200_OK);
    std::vector<std::thread> th;
    for (int k = 0; k < ncodecs; ++k) {
        if (share[k].empty()) continue;
        th.emplace_back([&, k]() {
            const std::vector<int>& idx = share[k];
            std::vector<lepb200_buffer> sub(idx.size());
            std::vector<lepb200_result> res(idx.size(), lepb200_result{nullptr, 0, 0});
            for (size_t q = 0; q < idx.size(); ++q) sub[q] = in[idx[q]];
            rcs[k] = compress ? lepb200_compress_jpegs(codecs[k], sub.data(), (int)sub.size(), res.data())
                              : lepb200_decompress_leps(codecs[k], sub.data(), (int)sub.size(), res.data());
            for (size_t q = 0; q < idx.size(); ++q) out[idx[q]] = res[q];        // data stays owned by codec k
        });
    }
    for (std::thread& t : th) t.join();
    for (int k = 0; k < ncodecs; ++k) if (rcs[k] != LEPB200_OK) return rcs[k];
    return LEPB200_OK;
}
}  // namespace

int lepb200_compress_jpegs_multi(lepb200_codec* const* codecs, int ncodecs, const lepb200_buffer* jpegs, int n, lepb200_result* out) {
    return run_multi(codecs, ncodecs, jpegs, n, out, true);
}
int lepb200_decompress_leps_multi(lepb200_codec* const* codecs, int ncodecs, const lepb200_buffer* leps, int n, lepb200_result* out) {
    return run_multi(codecs, ncodecs, leps, n, out, false);
}

// ---- staged host-only entry points (no GPU involved): parse + Huffman-decode one JPEG, expose its planes and
// thread-segment split as a lepb200_image, and assemble the .lep from externally coded segment streams.
struct lepb200_jpeg {
    Jpeg j;
    Splits sp;
    std::vector<std::vector<int16_t>> store;
    int16_t* planes[4] = {nullptr, nullptr, nullptr, nullptr};
    std::vector<uint8_t> out, hdr;
};

int lepb200_host_jpeg_open(const uint8_t* data, size_t len, lepb200_jpeg** out, int32_t* status) {
    return lepb200_host_jpeg_open_threads(data, len, 1, 8, out, status);
}

int lepb200_host_jpeg_open_threads(const uint8_t* data, size_t len, int min_threads, int max_threads, lepb200_jpeg** out, int32_t* status) {
    return lepb200_host_jpeg_open_split(data, len, min_threads, max_threads, 0, out, status);
}

int lepb200_host_jpeg_open_split(const uint8_t* data, size_t len, int min_threads, int max_threads, int even_split, lepb200_jpeg** out, int32_t* status) {
    return lepb200_host_jpeg_open_embedded(data, len, min_threads, max_threads, even_split, -1, 0, out, status);
}

int lepb200_host_jpeg_open_embedded(const uint8_t* data, size_t len, int min_threads, int max_threads, int even_split,
                                    long long embedding, int discard_meta, lepb200_jpeg** out, int32_t* status) {
    if (!out || !data) return LEPB200_ERR_INVALID;
    lepb200_jpeg* h = new lepb200_jpeg();
    *out = h;
    if (parse_jpeg(data, len, h->j, embedding < 0 ? -1 : embedding, discard_meta != 0)) {
        h->store.resize(h->j.ncmp);
        for (int c = 0; c < h->j.ncmp; ++c) {
            h->store[c].assign((size_t)h->j.cmp[c].bc * 64, 0);
            h->planes[c] = h->store[c].data();
        }
        if (decode_scans(h->j, h->planes)) h->sp = select_splits(h->j, (unsigned)std::max(max_threads, 1), (unsigned)std::max(min_threads, 1), even_split != 0);
    }
    if (status) *status = h->j.status;
    return LEPB200_OK;
}

const char* lepb200_host_jpeg_error(const lepb200_jpeg* h) { return h ? h->j.error.c_str() : "null"; }

int lepb200_host_jpeg_image(lepb200_jpeg* h, lepb200_image* img) {
    if (!h || !img || h->j.status) return LEPB200_ERR_INVALID;
    fill_image(*img, h->j, h->planes, h->sp.selected);
    return LEPB200_OK;
}

int lepb200_host_jpeg_scan(lepb200_jpeg* h, lepb200_jpeg_scan* sc) {
    if (!h || !sc || h->j.status) return LEPB200_ERR_INVALID;
    const Jpeg& j = h->j;
    GpuScanSetup gs;
    if (!gpu_scan_setup(j, gs)) return LEPB200_ERR_INVALID;
    fill_jpeg_scan(j, &gs, *sc);
    return LEPB200_OK;
}

int lepb200_host_jpeg_write_lep(lepb200_jpeg* h, const lepb200_stream* streams, int nseg, const uint8_t** data, size_t* len) {
    if (!h || !streams || !data || !len || h->j.status || nseg != (int)h->sp.selected.size()) return LEPB200_ERR_INVALID;
    std::vector<std::pair<const uint8_t*, size_t>> ss;
    for (int s = 0; s < nseg; ++s) ss.emplace_back(streams[s].data, (size_t)streams[s].len);
    std::string err;
    if (!write_lep(h->j, h->sp, ss, h->out, err)) { h->j.error = err; return LEPB200_ERR_INVALID; }
    *data = h->out.data();
    *len = h->out.size();
    return LEPB200_OK;
}

int lepb200_host_mux_plan(const size_t* lens, int nseg, lepb200_mux_packet* out, int cap) {
    if (!lens || nseg < 0 || nseg > 16 || (cap > 0 && !out)) return LEPB200_ERR_INVALID;
    std::vector<MuxPacket> plan;
    plan_mux(lens, nseg, plan);
    for (size_t k = 0; k < plan.size() && (int)k < cap; ++k) out[k] = plan[k];
    return (int)plan.size();
}

int lepb200_host_jpeg_header(lepb200_jpeg* h, const uint8_t** data, size_t* len) {
    if (!h || !data || !len || h->j.status) return LEPB200_ERR_INVALID;
    std::string err;
    if (!build_lep_header(h->j, h->sp, h->hdr, err)) { h->j.error = err; return LEPB200_ERR_INVALID; }
    *data = h->hdr.data();
    *len = h->hdr.size();
    return LEPB200_OK;
}

void lepb200_host_jpeg_close(lepb200_jpeg* h) { delete h; }

}  // extern "C"
