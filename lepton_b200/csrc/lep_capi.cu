// lep_capi.cu -- context, device memory management and the C ABI declared in include/lepton_b200.h.
// Single translation unit: the kernels are included so that nvcc sees one module (no -rdc needed).
#include <algorithm>
#include <cstdlib>
#include <cstdio>
#include <cstring>
#include <string>
#include <thread>
#include <tuple>
#include <vector>

#include <zlib.h>

#include "../../include/lepton_b200.h"
#include "lep_common.cuh"
#include "lep_predict.cuh"
#include "lep_encode.cu"
#include "lep_decode.cu"
#include "lep_decode_g2.cu"
#include "lep_huffpar.cu"
#include "lep_huffenc.cu"
#include "lep_mux.cu"
#include "lep_plan.cuh"
#include "lep_host.h"

using namespace lepb200;

namespace {

struct DevBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFree(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 4096;
        cudaError_t e = cudaMalloc(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFree(p); p = nullptr; cap = 0; }
    DevBuf() = default;
    DevBuf(const DevBuf&) = delete;
    DevBuf& operator=(const DevBuf&) = delete;
    ~DevBuf() { release(); }
};
struct HostBuf {
    void* p = nullptr;
    size_t cap = 0;
    cudaError_t reserve(size_t n) {
        if (n <= cap) return cudaSuccess;
        if (p) cudaFreeHost(p);
        p = nullptr; cap = 0;
        size_t want = n + n / 8 + 4096;
        cudaError_t e = cudaMallocHost(&p, want);
        if (e == cudaSuccess) cap = want;
        return e;
    }
    void release() { if (p) cudaFreeHost(p); p = nullptr; cap = 0; }
    HostBuf() = default;
    HostBuf(const HostBuf&) = delete;
    HostBuf& operator=(const HostBuf&) = delete;
    ~HostBuf() { release(); }
};

}  // namespace

struct lepb200_ctx {
    int device = 0;
    int sm_count = 0;
    cudaStream_t stream = nullptr;
    cudaEvent_t ev0 = nullptr, ev1 = nullptr, ev_mid = nullptr;
    std::string err;
    DevBuf d_planes, d_streams, d_tokens, d_dense, d_huff, d_hjobs, d_htabs, d_hrows, d_hpar, d_images, d_segs, d_order, d_counter, d_models, d_rows;
    DevBuf d_henc_out, d_henc_imgs, d_henc_segs, d_henc_tabs;
    DevBuf d_gather, d_lit;                // device container assembly: piece list, literal bytes (file headers + trailers)
    HostBuf h_lit;
    DevBuf d_rc_ck, d_rc_digits;           // parallel range coder: checkpoints of the range-only pass, deferred-carry digits
    DevBuf d_rc_ovf, d_rc_redo;            // streams longer than their slot (both range coder forms); serial form: segments it codes again
    HostBuf h_henc_out, h_henc_segs, h_henc_desc;
    cudaEvent_t status_ev = nullptr;       // parts mode: the D2H of the decode batch's segment records, queued ahead of the part copies
    bool status_queued = false;
    HuffEncodePlan henc;                  // jobs of the last Huffman encode (henc.off: where each image's scan bytes lie in the output buffers)
    // parts of the last lepb200_huffman_encode_resident_parts call: image range, segment range, byte range of the output,
    // the event behind the part's D2H copies on copy_stream
    struct HEncPart { int i0, i1, s0, s1; size_t b0, b1; cudaEvent_t done; };
    std::vector<HEncPart> henc_parts;
    std::vector<cudaEvent_t> part_events;      // pool: [2k] = part k's kernel, [2k + 1] = part k's copies
    cudaStream_t copy_stream = nullptr;        // D2H copies that run under the kernels of `stream`
    HostBuf h_segs, h_dense, h_stage, h_hjobs, h_hpar;
    size_t resident_plane_total = 0;
    int resident_images = 0;
    BatchPlan batch;                      // job tables of the current coder batch, device addresses once uploaded
    HuffDecodePlan hdec;                  // jobs of the last Huffman decode
    std::vector<int> rc_redo;             // serial range coder: segments it codes again
    int grid = 0;
    bool have_batch = false, launched = false, symbolised = false, is_encode = true;
    bool decode_fetched = false;          // h_segs holds the segment records of the current decode batch (lepb200_decode_fetch)
    float last_ms = -1.f, last_ms_a = -1.f, last_ms_huff = -1.f;
    uint64_t launches = 0;
    uint64_t alg_bytes = 0;
    uint64_t coded_blocks = 0;
    int enc_cta_cap = 0;                  // 0 = as many encode CTAs per SM as fit
    int huff_par = 1;                     // 1: images with enough entropy bytes take the many-threads-per-image kernels (lep_huffpar.cu)
    int huff_sub_bits = 0;                // bits per sub-sequence (one thread each); 0 = by batch size (LEPB200_HUFF_SUBSEQ_BITS overrides)
    int huff_par_iters = 0;               // synchronisation iterations of the last batch (diagnostic)
    int huff_redone = 0;                  // images of the last batch the sub-sequence kernels left to the serial walk (diagnostic)
    int huff_warps = 4;                   // images per CTA of the Huffman kernel
    int host_threads = 1;                 // host threads this context may use for staging copies
    int rc_feed = -1;                     // range pass token feed: 1 = cp.async ring in shared memory, 0 = register ring of plain loads, -1 = by
                                          // batch size: the ring up to 8192 segments, where the token feed bounds the chain; in larger
                                          // batches every SM streams and the feed stops mattering (not re-measured on the H100); LEPB200_RC_FEED
    int rc_mode = 1;                      // range coder: 1 = range-only pass + parallel pieces + carry pass (lep_rangepass / piece / norm kernels),
                                          // 0 = one serial chain per segment (lep_rangecode_kernel); LEPB200_RC_MODE
    int dec_mode = 0;                     // decode kernel: 0 = by batch size (group kernel when at least dec_group_min segments are in the
                                          // batch, else one warp per segment), 1 = always one warp per segment (lep_decode.cu),
                                          // 2 = always the group kernel (lep_decode_g2.cu)
    int dec_group_min = 6144;             // the group kernel carries 8 serial chains per warp: fewer instructions per decision, but a
                                          // longer latency per chain -- it wins when the chains alone fill the machine (measured on an
                                          // H100 SXM at a 400 W limit, 1080p 4:2:0 images: 8192 segments 999 ms against 1339 ms,
                                          // 6144 segments 936 ms against 1035 ms; 4096 segments 850 ms against 722 ms)
    int dec_threads_max = 16384;          // group kernel: segments per launch (one zero-filled 1.45 MB model each); more than a
                                          // decompress chunk of the file API holds, so that one launch covers a chunk
    int dec_lanes = 4;                    // group kernel: lanes per thread-segment, 32 / dec_lanes segments per warp in lock step
    int dec_group_grid = 0;               // group kernel: CTAs of the current batch
    int dec_threads = 0;                  // group kernel: model slots of the current batch (0: the batch uses the warp kernel)
    // decode batches with rANS-coded segments (lepb200_decode_upload_coded): they follow the bool-coded ones in the launch
    // order (BatchPlan::order_ans) and are decoded by launches of their own, group kernel or warp kernel by their own count
    int dec_threads_ans = 0, dec_group_grid_ans = 0, grid_ans = 0;
    bool stage_preuploaded = false;       // the caller pushed the staged scans itself (lepb200_huffman_stage_upload)
    bool canary = false;                  // batch of lepb200_encode_upload_tokens: stream and overflow arenas hold canary bytes
    size_t rc_ovf_used = 0;               // bytes of the overflow arena the last range coder run placed streams in
};

// lepb200_encode_upload_tokens / lepb200_encode_token_canaries: the byte the arenas are filled with, and how many of them
// follow every stream slot and the streams of the overflow arena
constexpr uint8_t CANARY_BYTE = 0xC3;
constexpr size_t CANARY_BYTES = 256;

#define CK(call)                                                                            \
    do {                                                                                    \
        cudaError_t e_ = (call);                                                            \
        if (e_ != cudaSuccess) {                                                            \
            ctx->err = std::string(#call) + ": " + cudaGetErrorString(e_);                  \
            return e_ == cudaErrorMemoryAllocation ? LEPB200_ERR_NOMEM : LEPB200_ERR_CUDA;  \
        }                                                                                   \
    } while (0)

namespace {

// lep_decode_g2_kernel<G>: launch shape (warps per CTA, thread-segments per warp) and resident CTAs per SM.  The groups'
// front regions take G2Cfg<G>::HOT_BYTES of dynamic shared memory (75 KB at G = 4: 32 groups of 2 400 bytes), more than the default 48 KB limit.
template <int G> cudaError_t group_kernel_allow_smem() {
    const cudaError_t e = cudaFuncSetAttribute(lep_decode_g2_kernel<G, G2Bool>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G2Cfg<G>::HOT_BYTES);
    return e != cudaSuccess ? e : cudaFuncSetAttribute(lep_decode_g2_kernel<G, G2Ans>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)G2Cfg<G>::HOT_BYTES);
}
template <int G> int group_ctas_per_sm() {
    int n = 0;
    if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&n, lep_decode_g2_kernel<G>, G2Cfg<G>::THREADS, G2Cfg<G>::HOT_BYTES) != cudaSuccess) n = 1;
    return std::max(n, 1);
}
void group_launch_shape(int lanes, int& warps, int& per_warp, int& ctas_per_sm) {
    per_warp = 32 / lanes;
    switch (lanes) {
    case 8: warps = G2Cfg<8>::WARPS; ctas_per_sm = group_ctas_per_sm<8>(); break;
    case 32: warps = G2Cfg<32>::WARPS; ctas_per_sm = group_ctas_per_sm<32>(); break;
    default: warps = G2Cfg<4>::WARPS; ctas_per_sm = group_ctas_per_sm<4>(); break;
    }
}
template <int G, class Coder = G2Bool> void launch_group_kernel(int grid, cudaStream_t st, const ImageDesc* images, SegDesc* segs, int first, int count, const int* order,
                                          int* counter, uint16_t* models, uint8_t* rows, size_t row_stride) {
    lep_decode_g2_kernel<G, Coder><<<grid, G2Cfg<G>::THREADS, G2Cfg<G>::HOT_BYTES, st>>>(images, segs, first, count, order, counter, models, rows, row_stride);
}

// The decode launches of one coder's segments, order[first .. first + n): the group kernel in launches of at most `threads`
// segments (threads > 0), else the warp kernel on a persistent grid of `wgrid` CTAs.
template <class WarpReader, class GroupCoder> int decode_launch_part(lepb200_ctx* ctx, int first, int n, int threads, int ggrid, int wgrid) {
    const ImageDesc* di = static_cast<const ImageDesc*>(ctx->d_images.p);
    SegDesc* ds = static_cast<SegDesc*>(ctx->d_segs.p);
    const int* dord = static_cast<const int*>(ctx->d_order.p);
    int* dcnt = static_cast<int*>(ctx->d_counter.p);
    uint16_t* dm = static_cast<uint16_t*>(ctx->d_models.p);
    uint8_t* dr = static_cast<uint8_t*>(ctx->d_rows.p);
    if (threads > 0) {
        // group kernel (lep_decode_g2.cu): G lanes per segment, 32 / G segments per warp in lock step; the groups of a
        // launch share a queue of at most dec_threads segments (one zero-filled model each), largest first
        int warps = 0, per_warp = 0, gsm = 0;
        group_launch_shape(ctx->dec_lanes, warps, per_warp, gsm);
        const int per_cta = warps * per_warp;
        for (int off = 0; off < n; off += threads) {
            const int count = std::min(threads, n - off);
            const int grid = std::max(1, std::min(ggrid, (count + per_cta - 1) / per_cta));
            CK(cudaMemsetAsync(ctx->d_models.p, 0, (size_t)count * MODEL_BYTES, ctx->stream));       // identity prior = zero fill
            CK(cudaMemsetAsync(ctx->d_counter.p, 0, sizeof(int), ctx->stream));
            switch (ctx->dec_lanes) {
            case 8: launch_group_kernel<8, GroupCoder>(grid, ctx->stream, di, ds, first + off, count, dord, dcnt, dm, dr, ctx->batch.row_stride); break;
            case 32: launch_group_kernel<32, GroupCoder>(grid, ctx->stream, di, ds, first + off, count, dord, dcnt, dm, dr, ctx->batch.row_stride); break;
            default: launch_group_kernel<4, GroupCoder>(grid, ctx->stream, di, ds, first + off, count, dord, dcnt, dm, dr, ctx->batch.row_stride); break;
            }
            CK(cudaGetLastError());
            ctx->launches += 1;
        }
    } else {
        if (first > 0) CK(cudaMemsetAsync(ctx->d_counter.p, 0, sizeof(int), ctx->stream));    // the batch's first queue: cleared before ev0
        lep_decode_kernel<WarpReader><<<wgrid, DEC_WARPS_PER_CTA * 32, 0, ctx->stream>>>(di, ds, n, dord + first, dcnt, dm, dr, ctx->batch.row_stride);
        CK(cudaGetLastError());
        ctx->launches += 1;
    }
    return LEPB200_OK;
}
// Common part of encode/decode upload: job tables (lep_plan.cuh), launch shape, pools, upload of the tables.
int build_batch(lepb200_ctx* ctx, const lepb200_image* images, int nimages, bool encode, const lepb200_stream* in,
                const uint8_t* coders = nullptr) {
    ctx->have_batch = false; ctx->launched = false; ctx->is_encode = encode; ctx->canary = false; ctx->decode_fetched = false;
    BatchPlan& b = ctx->batch;
    if (const char* e = plan_batch(b, images, nimages, encode, in, coders)) { ctx->err = e; return LEPB200_ERR_INVALID; }
    const int nseg = (int)b.segs.size();
    const int nbool = b.order_ans;                      // the bool-coded segments, launched before the rANS-coded ones

    // persistent grid: as many CTAs as can be resident, but no more warps than segments
    int per_sm = 0;
    if (encode) CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lep_encode_kernel<EncBool>, ENC_WARPS_PER_CTA * 32, 0));
    else CK(cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, lep_decode_kernel<BoolReader>, DEC_WARPS_PER_CTA * 32, 0));
    if (encode && ctx->enc_cta_cap > 0) per_sm = std::min(per_sm, ctx->enc_cta_cap);
    const int wpc = encode ? ENC_WARPS_PER_CTA : DEC_WARPS_PER_CTA;
    int grid = std::max(1, std::min(per_sm * ctx->sm_count, (nbool + wpc - 1) / wpc));
    ctx->grid = grid;
    ctx->grid_ans = std::max(1, std::min(per_sm * ctx->sm_count, (nseg - nbool + wpc - 1) / wpc));

    CK(ctx->d_planes.reserve(b.plane_total));
    CK(ctx->d_streams.reserve(b.stream_total + 256));
    CK(ctx->d_images.reserve(sizeof(ImageDesc) * nimages));
    CK(ctx->d_segs.reserve(sizeof(SegDesc) * nseg));
    CK(ctx->d_order.reserve(sizeof(int) * nseg));
    CK(ctx->d_counter.reserve(256));
    // decode kernel of each coder's segments: the group kernel when there are at least dec_group_min of them (one zero-filled
    // model per segment of a launch, one row buffer per resident group), else the warp kernel (one model and row buffer per warp)
    size_t model_bytes = 0, row_bytes = 0;
    auto part = [&](int n, int wgrid, int& threads, int& ggrid) {
        threads = 0;
        if (n == 0) return;
        const bool use_group = !encode && (ctx->dec_mode == 2 || (ctx->dec_mode == 0 && n >= ctx->dec_group_min));
        if (use_group) {
            threads = std::max(1, std::min(n, ctx->dec_threads_max));
            int warps = 0, per_warp = 0, gsm = 0;
            group_launch_shape(ctx->dec_lanes, warps, per_warp, gsm);
            const int per_cta = warps * per_warp;
            ggrid = std::max(1, std::min(gsm * ctx->sm_count, (threads + per_cta - 1) / per_cta));
            model_bytes = std::max(model_bytes, (size_t)threads * MODEL_BYTES);
            row_bytes = std::max(row_bytes, (size_t)ggrid * per_cta * b.row_stride);
        } else {
            model_bytes = std::max(model_bytes, (size_t)wgrid * wpc * MODEL_BYTES);
            row_bytes = std::max(row_bytes, (size_t)wgrid * wpc * b.row_stride);
        }
    };
    part(nbool, grid, ctx->dec_threads, ctx->dec_group_grid);
    part(nseg - nbool, ctx->grid_ans, ctx->dec_threads_ans, ctx->dec_group_grid_ans);
    CK(ctx->d_models.reserve(model_bytes));
    CK(ctx->d_rows.reserve(row_bytes));
    for (auto& d : b.images)
        for (int c = 0; c < d.ncmp; ++c) d.plane[c] += (unsigned long long)(uintptr_t)ctx->d_planes.p;
    for (auto& sd : b.segs) sd.stream += (unsigned long long)(uintptr_t)ctx->d_streams.p;
    CK(cudaMemcpyAsync(ctx->d_images.p, b.images.data(), sizeof(ImageDesc) * nimages, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_segs.p, b.segs.data(), sizeof(SegDesc) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_order.p, b.order.data(), sizeof(int) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    return 0;
}

// lep_compact_kernel for batches with rANS-coded segments: their streams lie in the token arena, 4-byte aligned (the rANS
// pass writes them backward from the end of the token slot), so the body moves 4-byte words
__global__ void lep_compact4_kernel(const SegDesc* __restrict__ segs, const unsigned long long* __restrict__ dst_off, uint8_t* __restrict__ dense, int nseg) {
    const int s = blockIdx.x;
    if (s >= nseg) return;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(segs[s].stream);
    uint8_t* dst = dense + dst_off[s];
    const uint32_t n = segs[s].status == 0 ? segs[s].len : 0;
    const uint32_t n4 = n / 4;
    const uint32_t* s4 = reinterpret_cast<const uint32_t*>(src);
    uint32_t* d4 = reinterpret_cast<uint32_t*>(dst);
    for (uint32_t i = threadIdx.x; i < n4; i += blockDim.x) d4[i] = s4[i];
    for (uint32_t i = n4 * 4 + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

__global__ void lep_compact_kernel(const SegDesc* __restrict__ segs, const unsigned long long* __restrict__ dst_off, uint8_t* __restrict__ dense, int nseg) {
    // one CTA per segment: copy the produced stream bytes into the dense output buffer (16-byte body, byte tails)
    const int s = blockIdx.x;
    if (s >= nseg) return;
    const uint8_t* src = reinterpret_cast<const uint8_t*>(segs[s].stream);
    uint8_t* dst = dense + dst_off[s];
    const uint32_t n = segs[s].status == 0 ? segs[s].len : 0;
    const uint32_t n16 = n / 16;           // src is 256-byte aligned, dst offsets are 16-byte aligned
    const uint4* s4 = reinterpret_cast<const uint4*>(src);
    uint4* d4 = reinterpret_cast<uint4*>(dst);
    for (uint32_t i = threadIdx.x; i < n16; i += blockDim.x) d4[i] = s4[i];
    for (uint32_t i = n16 * 16 + threadIdx.x; i < n; i += blockDim.x) dst[i] = src[i];
}

// Overflow arena of the range coder for `used` bytes of streams; in a canary batch it is filled with canary bytes first.
cudaError_t reserve_overflow(lepb200_ctx* ctx, size_t used) {
    ctx->rc_ovf_used = used;
    if (!ctx->canary) return ctx->d_rc_ovf.reserve(used);
    const cudaError_t e = ctx->d_rc_ovf.reserve(used + CANARY_BYTES);
    return e != cudaSuccess ? e : cudaMemsetAsync(ctx->d_rc_ovf.p, CANARY_BYTE, used + CANARY_BYTES, ctx->stream);
}

}  // namespace

extern "C" {

static int encode_prepass(lepb200_ctx* ctx);

int lepb200_device_available(void) {
    int n = 0;
    return cudaGetDeviceCount(&n) == cudaSuccess && n > 0;
}

size_t lepb200_model_bytes(void) { return MODEL_BYTES; }

int lepb200_create(lepb200_ctx** out, int device) {
    if (!out) return LEPB200_ERR_INVALID;
    *out = nullptr;
    int n = 0;
    if (cudaGetDeviceCount(&n) != cudaSuccess || n <= 0) return LEPB200_ERR_NO_DEVICE;
    if (device < 0 || device >= n) return LEPB200_ERR_INVALID;
    lepb200_ctx* ctx = new lepb200_ctx();
    ctx->device = device;
    if (cudaSetDevice(device) != cudaSuccess) { delete ctx; return LEPB200_ERR_CUDA; }
    cudaDeviceProp prop;
    if (cudaGetDeviceProperties(&prop, device) != cudaSuccess) { delete ctx; return LEPB200_ERR_CUDA; }
    ctx->sm_count = prop.multiProcessorCount;
    if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess || cudaStreamCreateWithFlags(&ctx->copy_stream, cudaStreamNonBlocking) != cudaSuccess ||
        cudaEventCreate(&ctx->ev0) != cudaSuccess ||
        cudaEventCreate(&ctx->ev1) != cudaSuccess || cudaEventCreate(&ctx->ev_mid) != cudaSuccess) {
        delete ctx;
        return LEPB200_ERR_CUDA;
    }
    if (cudaFuncSetAttribute(lep_rangepass_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RCT_SMEM_BYTES) != cudaSuccess ||
        cudaFuncSetAttribute(lep_rangepass_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)RCT_SMEM_TABLE_BYTES) != cudaSuccess ||
        group_kernel_allow_smem<4>() != cudaSuccess || group_kernel_allow_smem<8>() != cudaSuccess || group_kernel_allow_smem<32>() != cudaSuccess) {
        delete ctx;
        return LEPB200_ERR_CUDA;
    }
    if (const char* e = getenv("LEPB200_ENC_CTA_CAP")) ctx->enc_cta_cap = atoi(e);          // tuning overrides
    if (const char* e = getenv("LEPB200_HUFF_WARPS")) ctx->huff_warps = atoi(e);
    if (const char* e = getenv("LEPB200_HUFF_PAR")) ctx->huff_par = atoi(e);
    if (const char* e = getenv("LEPB200_HUFF_SUBSEQ_BITS")) ctx->huff_sub_bits = std::max(256, std::min(1 << 20, atoi(e))) & ~31;
    if (const char* e = getenv("LEPB200_DEC_MODE")) ctx->dec_mode = atoi(e);
    if (const char* e = getenv("LEPB200_RC_MODE")) ctx->rc_mode = atoi(e);
    if (const char* e = getenv("LEPB200_RC_FEED")) ctx->rc_feed = atoi(e);
    if (const char* e = getenv("LEPB200_DEC_THREADS")) ctx->dec_threads_max = std::max(32, atoi(e));
    if (const char* e = getenv("LEPB200_DEC_GROUP_MIN")) ctx->dec_group_min = std::max(1, atoi(e));
    if (const char* e = getenv("LEPB200_DEC_LANES")) {
        const int g = atoi(e);
        if (g == 4 || g == 8 || g == 32) ctx->dec_lanes = g;
    }
    *out = ctx;
    return LEPB200_OK;
}

void lepb200_set_encode_ctas_per_sm(lepb200_ctx* ctx, int n) { if (ctx && !getenv("LEPB200_ENC_CTA_CAP")) ctx->enc_cta_cap = n; }
void lepb200_set_host_threads(lepb200_ctx* ctx, int n) { if (ctx && n > 0) ctx->host_threads = n; }
void lepb200_set_huffman_warps_per_cta(lepb200_ctx* ctx, int n) { if (ctx && !getenv("LEPB200_HUFF_WARPS")) ctx->huff_warps = n; }

void lepb200_destroy(lepb200_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaEventDestroy(ctx->ev0);
    cudaEventDestroy(ctx->ev1);
    cudaEventDestroy(ctx->ev_mid);
    for (cudaEvent_t e : ctx->part_events) cudaEventDestroy(e);
    if (ctx->status_ev) cudaEventDestroy(ctx->status_ev);
    if (ctx->copy_stream) cudaStreamDestroy(ctx->copy_stream);
    cudaStreamDestroy(ctx->stream);
    delete ctx;                           // the buffers free themselves
}

void lepb200_release_device_buffers(lepb200_ctx* ctx) {
    if (!ctx) return;
    cudaSetDevice(ctx->device);
    cudaStreamSynchronize(ctx->stream);
    cudaStreamSynchronize(ctx->copy_stream);
    for (DevBuf* b : {&ctx->d_planes, &ctx->d_streams, &ctx->d_tokens, &ctx->d_dense, &ctx->d_huff, &ctx->d_hjobs, &ctx->d_htabs, &ctx->d_hrows,
                      &ctx->d_hpar, &ctx->d_images, &ctx->d_segs, &ctx->d_order, &ctx->d_counter, &ctx->d_models, &ctx->d_rows, &ctx->d_henc_out,
                      &ctx->d_henc_imgs, &ctx->d_henc_segs, &ctx->d_henc_tabs, &ctx->d_gather, &ctx->d_lit, &ctx->d_rc_ck, &ctx->d_rc_digits,
                      &ctx->d_rc_ovf, &ctx->d_rc_redo})
        b->release();
    ctx->have_batch = ctx->launched = ctx->decode_fetched = false;
}

const char* lepb200_last_error(const lepb200_ctx* ctx) { return ctx ? ctx->err.c_str() : "null context"; }
int lepb200_sync(lepb200_ctx* ctx) {
    if (!ctx) return LEPB200_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    CK(cudaStreamSynchronize(ctx->stream));
    return LEPB200_OK;
}
float lepb200_last_kernel_ms(lepb200_ctx* ctx) {
    if (!ctx) return -1.f;
    if (ctx->launched) {
        cudaSetDevice(ctx->device);
        float ms = -1.f;
        if (cudaEventSynchronize(ctx->ev1) == cudaSuccess && cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev1) == cudaSuccess) ctx->last_ms = ms;
        if (ctx->is_encode && cudaEventElapsedTime(&ms, ctx->ev0, ctx->ev_mid) == cudaSuccess) ctx->last_ms_a = ms;
    }
    return ctx->last_ms;
}
float lepb200_last_symbolise_ms(lepb200_ctx* ctx) {
    if (!ctx) return -1.f;
    lepb200_last_kernel_ms(ctx);
    return ctx->last_ms_a;
}
float lepb200_last_huffman_ms(lepb200_ctx* ctx) { return ctx ? ctx->last_ms_huff : -1.f; }
int lepb200_last_huffman_iterations(lepb200_ctx* ctx) { return ctx ? ctx->huff_par_iters : 0; }
int lepb200_last_huffman_redone(lepb200_ctx* ctx) { return ctx ? ctx->huff_redone : 0; }
uint64_t lepb200_kernel_launches(const lepb200_ctx* ctx) { return ctx ? ctx->launches : 0; }
uint64_t lepb200_last_algorithmic_bytes(const lepb200_ctx* ctx) { return ctx ? ctx->alg_bytes : 0; }

void* lepb200_pinned_alloc(size_t bytes) {
    void* p = nullptr;
    return cudaMallocHost(&p, bytes) == cudaSuccess ? p : nullptr;
}
void lepb200_pinned_free(void* p) { if (p) cudaFreeHost(p); }

// ------------------------------------------------------------------------------------------------ encode
int lepb200_encode_upload(lepb200_ctx* ctx, const lepb200_image* images, int nimages) {
    return lepb200_encode_upload_coded(ctx, images, nimages, nullptr);
}

int lepb200_encode_upload_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const uint8_t* coders) {
    if (!ctx) return LEPB200_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    int r = build_batch(ctx, images, nimages, true, nullptr, coders);
    if (r) return r;
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c)
            CK(cudaMemcpyAsync(reinterpret_cast<void*>(ctx->batch.images[i].plane[c]), images[i].planes[c], ctx->batch.plane_bytes[(size_t)i * 3 + c],
                               cudaMemcpyHostToDevice, ctx->stream));
    return encode_prepass(ctx);
}

static int encode_prepass(lepb200_ctx* ctx) {
    if (ctx->batch.tokens_known) {        // bounds came with the images (GPU Huffman decoder): nothing to count, nothing to wait for
        CK(ctx->d_tokens.reserve((size_t)ctx->batch.token_total * 2 + 256));
        ctx->have_batch = true;
        return LEPB200_OK;
    }
    // pre-pass: per-segment token upper bounds -> exact-fit token arena (sizes depend on the data, so one sync here)
    const int nseg = (int)ctx->batch.segs.size();
    lep_count_kernel<<<nseg, CNT_THREADS, 0, ctx->stream>>>(static_cast<const ImageDesc*>(ctx->d_images.p), static_cast<SegDesc*>(ctx->d_segs.p), nseg);
    CK(cudaGetLastError());
    unsigned long long* d_total = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctx->d_counter.p) + 64);
    lep_token_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(static_cast<SegDesc*>(ctx->d_segs.p), nseg, d_total);
    CK(cudaGetLastError());
    ctx->launches += 2;
    unsigned long long total_tokens = 0;
    CK(cudaMemcpyAsync(&total_tokens, d_total, sizeof(total_tokens), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(ctx->d_tokens.reserve((size_t)total_tokens * 2 + 256));
    ctx->batch.token_total = total_tokens;
    ctx->have_batch = true;
    return LEPB200_OK;
}

// ------------------------------------------------------------------------------------------------ GPU Huffman decode
uint8_t* lepb200_huffman_stage_reserve(lepb200_ctx* ctx, size_t bytes) {
    if (!ctx) return nullptr;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return nullptr;
    if (ctx->h_stage.reserve(bytes + 256) != cudaSuccess) { ctx->err = "pinned staging allocation failed"; return nullptr; }
    if (ctx->d_huff.reserve(bytes + 512) != cudaSuccess) { ctx->err = "device staging allocation failed"; return nullptr; }
    ctx->stage_preuploaded = false;
    return static_cast<uint8_t*>(ctx->h_stage.p);
}

// Asynchronous H2D of one staged range (callable from several host threads while others are still parsing); once used,
// the following lepb200_huffman_decode_to_device does not copy the staging buffer again, so ALL scans must be pushed.
int lepb200_huffman_stage_upload(lepb200_ctx* ctx, size_t offset, size_t bytes) {
    if (!ctx || !ctx->h_stage.p || offset + bytes > ctx->h_stage.cap || offset + bytes > ctx->d_huff.cap) return LEPB200_ERR_INVALID;
    if (cudaSetDevice(ctx->device) != cudaSuccess) return LEPB200_ERR_CUDA;
    ctx->stage_preuploaded = true;
    if (cudaMemcpyAsync(static_cast<uint8_t*>(ctx->d_huff.p) + offset, static_cast<uint8_t*>(ctx->h_stage.p) + offset, bytes,
                        cudaMemcpyHostToDevice, ctx->stream) != cudaSuccess) return LEPB200_ERR_CUDA;
    return LEPB200_OK;
}

int lepb200_huffman_decode_to_device(lepb200_ctx* ctx, lepb200_jpeg_scan* scans, int n) {
    if (!ctx || !scans || n <= 0) return LEPB200_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    ctx->have_batch = false; ctx->launched = false; ctx->decode_fetched = false; ctx->resident_images = 0;
    // sub-sequence length of the many-threads-per-image kernels: longer sub-sequences need fewer synchronisation passes
    // (8192 bits: 3, 4096: 5, 2048: 9 on 1080p files), as long as the batch still gives every SM its 2048 threads
    int sub_bits = ctx->huff_sub_bits;
    if (sub_bits <= 0) {
        uint64_t bits = 0;
        for (int i = 0; i < n; ++i) if (scans[i].entropy && scans[i].ncmp > 1 && scans[i].rsti == 0) bits += (uint64_t)scans[i].nbytes * 8;
        sub_bits = 2048;
        for (int cand : {16384, 8192, 4096}) if (bits / (uint64_t)cand >= (uint64_t)ctx->sm_count * 2048) { sub_bits = cand; break; }
    }
    // in-place mode: the caller de-stuffed straight into this context's pinned staging buffer
    // (lepb200_huffman_stage_reserve), 16-byte aligned with >= 16 spare bytes after each scan -> no gather copy
    HuffDecodePlan& p = ctx->hdec;
    if (const char* e = plan_huffman_decode(p, scans, n, ctx->huff_par != 0, sub_bits, static_cast<const uint8_t*>(ctx->h_stage.p), ctx->h_stage.cap)) {
        ctx->err = e;
        return LEPB200_ERR_INVALID;
    }
    std::vector<HuffJob>& jobs = p.jobs;
    const std::vector<HuffTableDev>& tabs = p.tabs.tabs;
    const size_t plane_total = p.plane_total, huff_total = p.huff_total, rows_total = p.rows_total;
    const uint32_t sub_total = p.sub_total;
    CK(ctx->d_planes.reserve(plane_total + 256));
    CK(ctx->d_huff.reserve(huff_total + 256));
    CK(ctx->d_hrows.reserve(rows_total + 256));
    CK(ctx->d_htabs.reserve(sizeof(HuffTableDev) * std::max<size_t>(1, tabs.size())));
    if (!p.in_place) CK(ctx->h_stage.reserve(huff_total + 256));
    uint8_t* hs = static_cast<uint8_t*>(ctx->h_stage.p);
    if (p.in_place) {
        if (!ctx->stage_preuploaded)          // (a caller that uploads itself has zeroed the 16 bytes behind each scan)
            for (int i = 0; i < n; ++i) if (scans[i].entropy) memset(hs + jobs[i].huff + scans[i].nbytes, 0, 16);   // the decoder reads whole words past the end
    } else {
        // gather the de-stuffed scans into the pinned staging buffer (hundreds of MB per chunk): split over host threads
        const int nt = std::max(1, std::min(ctx->host_threads, n));
        auto copy_range = [&](int t) {
            for (int i = t; i < n; i += nt) {
                const HuffJob& jb = jobs[i];
                if (!scans[i].entropy) continue;
                memcpy(hs + jb.huff, scans[i].entropy, scans[i].nbytes);
                memset(hs + jb.huff + scans[i].nbytes, 0, align_up((size_t)scans[i].nbytes + 16, 16) - scans[i].nbytes);
            }
        };
        if (nt == 1) copy_range(0);
        else {
            std::vector<std::thread> th;
            for (int t = 0; t < nt; ++t) th.emplace_back(copy_range, t);
            for (auto& t : th) t.join();
        }
    }
    const unsigned long long d_rows = (unsigned long long)(uintptr_t)ctx->d_hrows.p;
    for (HuffJob& jb : jobs) {
        jb.huff += (unsigned long long)(uintptr_t)ctx->d_huff.p;
        jb.rows += d_rows;
        for (int c = 0; c < jb.ncmp; ++c) jb.plane[c] += (unsigned long long)(uintptr_t)ctx->d_planes.p;
    }
    CK(ctx->d_hjobs.reserve(align_up(sizeof(HuffJob) * n, 256)));
    CK(cudaMemsetAsync(ctx->d_planes.p, 0, plane_total, ctx->stream));
    if (!(p.in_place && ctx->stage_preuploaded)) CK(cudaMemcpyAsync(ctx->d_huff.p, hs, huff_total, cudaMemcpyHostToDevice, ctx->stream));
    ctx->stage_preuploaded = false;
    CK(cudaMemcpyAsync(ctx->d_hjobs.p, jobs.data(), sizeof(HuffJob) * n, cudaMemcpyHostToDevice, ctx->stream));

    if (!tabs.empty()) CK(cudaMemcpyAsync(ctx->d_htabs.p, tabs.data(), sizeof(HuffTableDev) * tabs.size(), cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    // CTA width: 7 images per CTA puts a 1024-image chunk on one CTA per SM, whose registers fit next to the encode
    // kernel of the previous chunk when that one is capped (lepb200_set_encode_ctas_per_sm), so the two overlap
    ctx->huff_par_iters = 0;
    if (sub_total > 0) {
        // sub-sequence kernels (lep_huffpar.cu): arrays of 32 bytes per sub-sequence, then sub_base and the dirty counters
        constexpr int ITER_CAP = 62;
        const size_t o_exit = 0, o_cnt = align_up((size_t)sub_total * 8, 256), o_tok = o_cnt + align_up((size_t)sub_total * 16, 256),
                     o_epoch = o_tok + align_up((size_t)sub_total * 4, 256), o_dirty = o_epoch + align_up((size_t)sub_total * 4, 256),
                     o_base = o_dirty + 256, o_end = o_base + align_up(((size_t)n + 1) * 4, 256);
        CK(ctx->d_hpar.reserve(o_end));
        uint8_t* hp = static_cast<uint8_t*>(ctx->d_hpar.p);
        CK(cudaMemsetAsync(hp + o_epoch, 0, o_base - o_epoch, ctx->stream));
        CK(ctx->h_hpar.reserve(align_up(((size_t)n + 1) * 4, 256) + 256));
        uint32_t* h_base = static_cast<uint32_t*>(ctx->h_hpar.p);
        unsigned int* h_dirty = reinterpret_cast<unsigned int*>(static_cast<uint8_t*>(ctx->h_hpar.p) + align_up(((size_t)n + 1) * 4, 256));
        memcpy(h_base, p.sub_base.data(), ((size_t)n + 1) * 4);
        CK(cudaMemcpyAsync(hp + o_base, h_base, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, ctx->stream));
        HpArrays a;
        a.exit = reinterpret_cast<unsigned long long*>(hp + o_exit); a.cnt = reinterpret_cast<uint4*>(hp + o_cnt);
        a.tok = reinterpret_cast<uint32_t*>(hp + o_tok); a.epoch = reinterpret_cast<uint32_t*>(hp + o_epoch);
        a.sub_base = reinterpret_cast<const uint32_t*>(hp + o_base); a.total = sub_total; a.sub_bits = (uint32_t)sub_bits;
        unsigned int* d_dirty = reinterpret_cast<unsigned int*>(hp + o_dirty);
        HuffJob* dj = static_cast<HuffJob*>(ctx->d_hjobs.p);
        const HuffTableDev* dt = static_cast<const HuffTableDev*>(ctx->d_htabs.p);
        const unsigned grid = (sub_total + HP_THREADS - 1) / HP_THREADS;
        int iter = 0;
        auto sync_iter = [&]() {
            lep_huffpar_sync_kernel<<<grid, HP_THREADS, 0, ctx->stream>>>(dj, n, dt, (int)tabs.size(), a, iter, ITER_CAP, d_dirty);
            ++iter; ctx->launches += 1;
        };
        sync_iter(); sync_iter(); sync_iter();
        for (;;) {              // until no sub-sequence has to run again (dirty[k] = sub-sequences that iteration k has to decode)
            CK(cudaMemcpyAsync(h_dirty, d_dirty, 64 * sizeof(unsigned int), cudaMemcpyDeviceToHost, ctx->stream));
            CK(cudaStreamSynchronize(ctx->stream));
            if (iter > ITER_CAP || h_dirty[iter] == 0) break;
            sync_iter();
            if (iter <= ITER_CAP) sync_iter();
        }
        ctx->huff_par_iters = iter;
        lep_huffpar_prefix_kernel<<<(n + 127) / 128, 128, 0, ctx->stream>>>(dj, n, a);
        lep_huffpar_write_kernel<<<grid, HP_THREADS, 0, ctx->stream>>>(dj, n, dt, (int)tabs.size(), a);
        ctx->launches += 2;
        CK(cudaGetLastError());
    }
    // the serial walk: every image the kernels above did not take or did not finish cleanly
    const int hw = std::max(1, std::min(HUFF_MAX_WARPS, ctx->huff_warps));
    lep_huffdecode_kernel<<<(n + hw - 1) / hw, hw * 32, 0, ctx->stream>>>(
        static_cast<HuffJob*>(ctx->d_hjobs.p), n, static_cast<const HuffTableDev*>(ctx->d_htabs.p), (int)tabs.size());
    CK(cudaGetLastError());
    CK(cudaEventRecord(ctx->ev_mid, ctx->stream));
    ctx->launches += 1;
    CK(ctx->h_hjobs.reserve(sizeof(HuffJob) * n + rows_total));
    HuffJob* hj = static_cast<HuffJob*>(ctx->h_hjobs.p);
    uint8_t* hrows = reinterpret_cast<uint8_t*>(hj + n);
    CK(cudaMemcpyAsync(hj, ctx->d_hjobs.p, sizeof(HuffJob) * n, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(hrows, ctx->d_hrows.p, rows_total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    cudaEventElapsedTime(&ctx->last_ms_huff, ctx->ev0, ctx->ev_mid);
    ctx->huff_redone = 0;
    for (int i = 0; i < n; ++i) ctx->huff_redone += hj[i].nsub != 0 && !(hj[i].par_done && !hj[i].par_redo);
    huffman_decode_results(scans, n, hj, hrows, d_rows);
    ctx->resident_plane_total = plane_total;
    ctx->resident_images = n;
    return LEPB200_OK;
}

int lepb200_encode_upload_resident(lepb200_ctx* ctx, const lepb200_image* images, int nimages) {
    if (!ctx) return LEPB200_ERR_INVALID;
    if (ctx->resident_images != nimages) { ctx->err = "encode_upload_resident: no matching huffman_decode_to_device batch"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    // resident images carry no host planes (validate_image wants non-null pointers); placeholder images do
    std::vector<lepb200_image> tmp(images, images + nimages);
    for (auto& im : tmp) for (int c = 0; c < im.ncmp && c < 3; ++c) if (!im.planes[c]) im.planes[c] = reinterpret_cast<int16_t*>(uintptr_t(1));
    void* const planes_before = ctx->d_planes.p;
    int r = build_batch(ctx, tmp.data(), nimages, true, nullptr);
    if (r) return r;
    if (ctx->d_planes.p != planes_before) { ctx->err = "encode_upload_resident: plane arena moved (geometry mismatch)"; return LEPB200_ERR_INVALID; }
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp && c < 3; ++c)
            if (images[i].planes[c])
                CK(cudaMemcpyAsync(reinterpret_cast<void*>(ctx->batch.images[i].plane[c]), images[i].planes[c], ctx->batch.plane_bytes[(size_t)i * 3 + c],
                                   cudaMemcpyHostToDevice, ctx->stream));
    ctx->resident_images = 0;
    return encode_prepass(ctx);
}

int lepb200_encode_launch_symbolise(lepb200_ctx* ctx) {
    if (!ctx || !ctx->have_batch || !ctx->is_encode) { if (ctx) ctx->err = "encode_launch without encode_upload"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size(), nbool = ctx->batch.order_ans;
    // one launch per coder: the bool-coded segments (order[0 .. nbool)), then the rANS-coded ones, each with its own queue
    // (the rANS part's work counter sits 32 bytes into the counter buffer)
    int* dcnt = static_cast<int*>(ctx->d_counter.p);
    CK(cudaMemsetAsync(ctx->d_counter.p, 0, nbool < nseg ? 64 : sizeof(int), ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    const ImageDesc* di = static_cast<const ImageDesc*>(ctx->d_images.p);
    SegDesc* ds = static_cast<SegDesc*>(ctx->d_segs.p);
    const int* dord = static_cast<const int*>(ctx->d_order.p);
    uint16_t* dm = static_cast<uint16_t*>(ctx->d_models.p);
    uint8_t* dr = static_cast<uint8_t*>(ctx->d_rows.p);
    uint16_t* dt = static_cast<uint16_t*>(ctx->d_tokens.p);
    if (nbool > 0) {
        lep_encode_kernel<EncBool><<<ctx->grid, ENC_WARPS_PER_CTA * 32, 0, ctx->stream>>>(di, ds, nbool, dord, dcnt, dm, dr, ctx->batch.row_stride, dt);
        CK(cudaGetLastError());
        ctx->launches += 1;
    }
    if (nbool < nseg) {
        lep_encode_kernel<EncAns><<<ctx->grid_ans, ENC_WARPS_PER_CTA * 32, 0, ctx->stream>>>(di, ds, nseg - nbool, dord + nbool, dcnt + 8, dm, dr,
                                                                                               ctx->batch.row_stride, dt);
        CK(cudaGetLastError());
        ctx->launches += 1;
    }
    CK(cudaEventRecord(ctx->ev_mid, ctx->stream));
    ctx->symbolised = true;
    return LEPB200_OK;
}

int lepb200_encode_launch_rangecode(lepb200_ctx* ctx) {
    if (!ctx || !ctx->symbolised || !ctx->is_encode) { if (ctx) ctx->err = "encode_launch_rangecode without encode_launch_symbolise"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    // the bool-coded segments are segs[0 .. nbool) and order[0 .. nbool) (plan_batch): the range coder takes those, the
    // rANS pass the others, in every rc_mode
    const int nall = (int)ctx->batch.segs.size(), nseg = ctx->batch.order_ans;
    ctx->rc_ovf_used = 0;
    if (nseg == 0) {
        // no bool-coded segment
    } else if (ctx->rc_mode == 1) {
        // range-only pass -> digit layout (one small D2H + sync: the arena size depends on the data) -> parallel pieces -> carries
        SegDesc* ds = static_cast<SegDesc*>(ctx->d_segs.p);
        const int* dord = static_cast<const int*>(ctx->d_order.p);
        const uint16_t* dtok = static_cast<const uint16_t*>(ctx->d_tokens.p);
        CK(ctx->d_rc_ck.reserve(rc_checkpoints(ctx->batch.token_total, nseg) * sizeof(unsigned long long)));
        unsigned long long* dck = static_cast<unsigned long long*>(ctx->d_rc_ck.p);
        const bool trace = getenv("LEPB200_TRACE") != nullptr;           // per-kernel times on stderr (diagnostics; adds a sync)
        cudaEvent_t te[4] = {nullptr, nullptr, nullptr, nullptr};
        if (trace) { for (auto& e : te) cudaEventCreate(&e); cudaEventRecord(te[0], ctx->stream); }
        const bool async_feed = ctx->rc_feed < 0 ? nseg <= 8192 : ctx->rc_feed != 0;
        if (async_feed) lep_rangepass_kernel<true><<<(nseg + RCT_THREADS - 1) / RCT_THREADS, RCT_THREADS, RCT_SMEM_BYTES, ctx->stream>>>(ds, nseg, dord, dtok, dck);
        else lep_rangepass_kernel<false><<<(nseg + RCT_THREADS - 1) / RCT_THREADS, RCT_THREADS, RCT_SMEM_TABLE_BYTES, ctx->stream>>>(ds, nseg, dord, dtok, dck);
        CK(cudaGetLastError());
        unsigned long long* d_total = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctx->d_counter.p) + 128);
        lep_digit_offsets_kernel<<<1, 1024, 0, ctx->stream>>>(ds, nseg, d_total, d_total + 1);
        CK(cudaGetLastError());
        // [0] digits, [1] bytes of the overflow arena (streams longer than their slot; 0 for photo batches) -- one copy, one sync
        unsigned long long totals[2] = {0, 0};
        CK(cudaMemcpyAsync(totals, d_total, sizeof(totals), cudaMemcpyDeviceToHost, ctx->stream));
        CK(cudaStreamSynchronize(ctx->stream));
        const unsigned long long total_digits = totals[0];
        if (totals[1]) CK(reserve_overflow(ctx, (size_t)totals[1]));
        if (trace) cudaEventRecord(te[1], ctx->stream);
        CK(ctx->d_rc_digits.reserve((size_t)total_digits * 4 + 256));
        CK(cudaMemsetAsync(ctx->d_rc_digits.p, 0, (size_t)total_digits * 4, ctx->stream));
        uint32_t* ddig = static_cast<uint32_t*>(ctx->d_rc_digits.p);
        lep_rangepiece_kernel<<<dim3(8, (unsigned)nseg), RCP_THREADS, 0, ctx->stream>>>(ds, nseg, dtok, dck, ddig);
        CK(cudaGetLastError());
        if (trace) cudaEventRecord(te[2], ctx->stream);
        lep_rangenorm_kernel<<<(nseg + RCN_WARPS - 1) / RCN_WARPS, RCN_WARPS * 32, 0, ctx->stream>>>(ds, nseg, dord, ddig,
                                                                                                       static_cast<uint8_t*>(ctx->d_rc_ovf.p));
        CK(cudaGetLastError());
        if (trace) {
            cudaEventRecord(te[3], ctx->stream);
            cudaEventSynchronize(te[3]);
            float a = 0, b = 0, c = 0;
            cudaEventElapsedTime(&a, te[0], te[1]); cudaEventElapsedTime(&b, te[1], te[2]); cudaEventElapsedTime(&c, te[2], te[3]);
            fprintf(stderr, "[trace]   range coder: range pass + offsets %.1f ms, pieces (incl. digit zero fill) %.1f ms, carries %.1f ms, %d segments\n", a, b, c, nseg);
            for (auto& e : te) cudaEventDestroy(e);
        }
        ctx->launches += 4;
    } else {
        lep_rangecode_kernel<<<(nseg + RC_THREADS - 1) / RC_THREADS, RC_THREADS, 0, ctx->stream>>>(
            static_cast<SegDesc*>(ctx->d_segs.p), nseg, static_cast<const int*>(ctx->d_order.p), static_cast<const uint16_t*>(ctx->d_tokens.p));
        CK(cudaGetLastError());
        ctx->launches += 1;
    }
    if (nall > nseg) {
        // rANS pass (lep_encode.cu): one thread per segment, the stream written in place into the segment's token slot
        const int n = nall - nseg;
        lep_anspass_kernel<<<(n + ANS_THREADS - 1) / ANS_THREADS, ANS_THREADS, 0, ctx->stream>>>(
            static_cast<SegDesc*>(ctx->d_segs.p), n, static_cast<const int*>(ctx->d_order.p) + nseg, static_cast<uint16_t*>(ctx->d_tokens.p));
        CK(cudaGetLastError());
        ctx->launches += 1;
    }
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->symbolised = false;
    ctx->launched = true;
    return LEPB200_OK;
}

int lepb200_encode_launch(lepb200_ctx* ctx) {
    const int r = lepb200_encode_launch_symbolise(ctx);
    return r ? r : lepb200_encode_launch_rangecode(ctx);
}

// Serial range coder (rc_mode 0): codes the segments whose stream outgrew its slot again, into the overflow arena
// (plan_serial_rerun).  hs (the segment records, fetched) is updated in place.
static int rerun_overflowed_serial(lepb200_ctx* ctx, SegDesc* hs, int nseg) {
    if (ctx->rc_mode == 1) return LEPB200_OK;
    std::vector<int>& redo = ctx->rc_redo;
    const size_t total = plan_serial_rerun(hs, ctx->batch.order_ans, redo);       // the bool-coded segments, segs[0 .. order_ans)
    if (redo.empty()) return LEPB200_OK;
    CK(reserve_overflow(ctx, total));
    CK(ctx->d_rc_redo.reserve(sizeof(int) * redo.size()));
    for (int s : redo) hs[s].stream += (unsigned long long)(uintptr_t)ctx->d_rc_ovf.p;
    const int n = (int)redo.size();
    CK(cudaMemcpyAsync(ctx->d_segs.p, hs, sizeof(SegDesc) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_rc_redo.p, redo.data(), sizeof(int) * n, cudaMemcpyHostToDevice, ctx->stream));
    lep_rangecode_kernel<<<(n + RC_THREADS - 1) / RC_THREADS, RC_THREADS, 0, ctx->stream>>>(
        static_cast<SegDesc*>(ctx->d_segs.p), n, static_cast<const int*>(ctx->d_rc_redo.p), static_cast<const uint16_t*>(ctx->d_tokens.p));
    CK(cudaGetLastError());
    ctx->launches += 1;
    CK(cudaMemcpyAsync(hs, ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    return LEPB200_OK;
}

int lepb200_encode_fetch(lepb200_ctx* ctx, lepb200_stream* out) {
    if (!ctx || !ctx->launched || !ctx->is_encode || !out) { if (ctx) ctx->err = "encode_fetch without encode_launch"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size();
    CK(ctx->h_segs.reserve(sizeof(SegDesc) * nseg + sizeof(unsigned long long) * nseg));
    SegDesc* hs = static_cast<SegDesc*>(ctx->h_segs.p);
    CK(cudaMemcpyAsync(hs, ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    if (const int r = rerun_overflowed_serial(ctx, hs, nseg)) return r;
    // dense layout of the produced streams
    unsigned long long* offs = reinterpret_cast<unsigned long long*>(hs + nseg);
    size_t total = 0;
    uint64_t alg = 0;
    for (int s = 0; s < nseg; ++s) {
        offs[s] = total;
        size_t n = hs[s].status == 0 ? hs[s].len : 0;
        total += align_up(n, 16);
        alg += (uint64_t)ctx->batch.seg_blocks[s] * 128 + n;
    }
    ctx->alg_bytes = alg;
    const size_t dense_bytes = align_up(total, 256);
    CK(ctx->d_dense.reserve(dense_bytes + sizeof(unsigned long long) * nseg));
    CK(ctx->h_dense.reserve(total + 16));
    unsigned long long* d_offs = reinterpret_cast<unsigned long long*>(static_cast<uint8_t*>(ctx->d_dense.p) + dense_bytes);
    CK(cudaMemcpyAsync(d_offs, offs, sizeof(unsigned long long) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    if (ctx->batch.order_ans == nseg)
        lep_compact_kernel<<<nseg, 256, 0, ctx->stream>>>(static_cast<const SegDesc*>(ctx->d_segs.p), d_offs, static_cast<uint8_t*>(ctx->d_dense.p), nseg);
    else
        lep_compact4_kernel<<<nseg, 256, 0, ctx->stream>>>(static_cast<const SegDesc*>(ctx->d_segs.p), d_offs, static_cast<uint8_t*>(ctx->d_dense.p), nseg);
    CK(cudaGetLastError());
    ctx->launches += 1;
    if (total) CK(cudaMemcpyAsync(ctx->h_dense.p, ctx->d_dense.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const std::vector<int>& seg_out = ctx->batch.seg_out;          // the caller's order of the segments (plan_batch)
    for (int s = 0; s < nseg; ++s) {
        lepb200_stream& o = out[seg_out.empty() ? s : seg_out[s]];
        o.data = static_cast<const uint8_t*>(ctx->h_dense.p) + offs[s];
        o.len = hs[s].status == 0 ? hs[s].len : 0;
        o.status = hs[s].status;
        o.reserved = 0;
        o.ndecisions = (uint64_t)hs[s].ndecisions_lo | ((uint64_t)hs[s].ndecisions_hi << 32);
    }
    return LEPB200_OK;
}

// Final .lep files from the device (SURVEY.md section 8(f) row 3): headers[i] = everything in front of the mux packets
// of image i (fixed header + zlib'd JPEG header + "CMP", built on the host: lephost::build_lep_header); the MuxWriter
// schedule is planned on the host from the stream lengths the range coder reports (lephost::plan_mux, data-free), the
// bytes are moved by lep_gather_kernel, the LE32 size trailer (vp8_encoder.cc:603-614) is a literal.
int lepb200_encode_fetch_files(lepb200_ctx* ctx, const lepb200_buffer* headers, lepb200_result* files) {
    if (!ctx || !ctx->launched || !ctx->is_encode || !headers || !files) { if (ctx) ctx->err = "encode_fetch_files without encode_launch"; return LEPB200_ERR_INVALID; }
    if (ctx->batch.order_ans != (int)ctx->batch.segs.size()) {
        ctx->err = "encode_fetch_files: rANS-coded segments (container version 3) have no device file writer; fetch them with encode_fetch";
        return LEPB200_ERR_INVALID;
    }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size(), nimg = (int)ctx->batch.images.size();
    CK(ctx->h_segs.reserve(sizeof(SegDesc) * nseg));
    SegDesc* hs = static_cast<SegDesc*>(ctx->h_segs.p);
    CK(cudaMemcpyAsync(hs, ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    if (const int r = rerun_overflowed_serial(ctx, hs, nseg)) return r;
    // literals: header + 4 trailer bytes per image, 16-byte aligned
    size_t lit_total = 0;
    std::vector<size_t> lit_off(nimg);
    for (int i = 0; i < nimg; ++i) { lit_off[i] = lit_total; lit_total += align_up(headers[i].len + 4, 16); }
    CK(ctx->h_lit.reserve(lit_total + 64));
    CK(ctx->d_lit.reserve(lit_total + 256));
    uint8_t* hl = static_cast<uint8_t*>(ctx->h_lit.p);
    const unsigned long long dl = (unsigned long long)(uintptr_t)ctx->d_lit.p;
    std::vector<GatherPiece> pieces;
    pieces.reserve((size_t)nseg * 32 + 2 * (size_t)nimg);
    std::vector<size_t> file_off(nimg, 0);
    std::vector<lephost::MuxPacket> plan;
    size_t total = 0;
    uint64_t alg = 0;
    int s0 = 0;
    for (int i = 0; i < nimg; ++i) {
        int s1 = s0;
        while (s1 < nseg && hs[s1].image == i) ++s1;
        int st = 0;
        size_t lens[LEPB200_MAX_SEGMENTS];
        const int ns = s1 - s0;
        for (int s = s0; s < s1; ++s) {
            if (hs[s].status && !st) st = hs[s].status;
            if (s - s0 < LEPB200_MAX_SEGMENTS) lens[s - s0] = hs[s].len;
            alg += (uint64_t)ctx->batch.seg_blocks[s] * 128 + (hs[s].status == 0 ? hs[s].len : 0);
        }
        files[i].data = nullptr; files[i].len = 0; files[i].status = st;
        if (st == 0 && (ns < 1 || ns > LEPB200_MAX_SEGMENTS || !headers[i].data || headers[i].len == 0)) files[i].status = st = LEPB200_ST_NOT_HANDLED;
        if (st == 0) {
            lephost::plan_mux(lens, ns, plan);
            total = align_up(total, 16);
            file_off[i] = total;
            memcpy(hl + lit_off[i], headers[i].data, headers[i].len);
            unsigned long long saddr[LEPB200_MAX_SEGMENTS];
            for (int k = 0; k < ns; ++k) saddr[k] = hs[s0 + k].stream;
            const uint32_t fsz = gather_file_pieces(plan.data(), plan.size(), saddr, dl + lit_off[i], hl + lit_off[i], headers[i].len, total, pieces);
            files[i].len = fsz;
            total += fsz;
        }
        s0 = s1;
    }
    ctx->alg_bytes = alg;
    if (pieces.empty()) return LEPB200_OK;
    CK(ctx->d_dense.reserve(total + 256));
    CK(ctx->h_dense.reserve(total + 16));
    CK(ctx->d_gather.reserve(sizeof(GatherPiece) * pieces.size()));
    CK(cudaMemcpyAsync(ctx->d_lit.p, hl, lit_total, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_gather.p, pieces.data(), sizeof(GatherPiece) * pieces.size(), cudaMemcpyHostToDevice, ctx->stream));
    const unsigned grid = (unsigned)std::min<size_t>((pieces.size() + GATHER_WARPS - 1) / GATHER_WARPS, (size_t)ctx->sm_count * 8);
    lep_gather_kernel<<<grid, GATHER_WARPS * 32, 0, ctx->stream>>>(static_cast<const GatherPiece*>(ctx->d_gather.p), (uint32_t)pieces.size(), static_cast<uint8_t*>(ctx->d_dense.p));
    CK(cudaGetLastError());
    ctx->launches += 1;
    CK(cudaMemcpyAsync(ctx->h_dense.p, ctx->d_dense.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    for (int i = 0; i < nimg; ++i) if (files[i].status == 0) files[i].data = static_cast<const uint8_t*>(ctx->h_dense.p) + file_off[i];
    return LEPB200_OK;
}

int lepb200_encode_images(lepb200_ctx* ctx, const lepb200_image* images, int nimages, lepb200_stream* out) {
    return lepb200_encode_images_coded(ctx, images, nimages, nullptr, out);
}

int lepb200_encode_images_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const uint8_t* coders, lepb200_stream* out) {
    int r = lepb200_encode_upload_coded(ctx, images, nimages, coders);
    if (r) return r;
    r = lepb200_encode_launch(ctx);
    if (r) return r;
    return lepb200_encode_fetch(ctx, out);
}

// An encode batch as kernel A leaves it, from caller token streams: token slots as lep_token_offsets_kernel lays them out,
// stream slots of caps[s] bytes each followed by CANARY_BYTES canary bytes, longest streams first.  Segments are grouped
// into nfiles files (consecutive, seg_per_file[f] each) for lepb200_encode_fetch_files.
int lepb200_encode_upload_tokens(lepb200_ctx* ctx, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* caps, int nseg,
                                 const int32_t* seg_per_file, int nfiles) {
    return lepb200_encode_upload_tokens_coded(ctx, tokens, ntok, caps, nseg, seg_per_file, nfiles, nullptr);
}

// coders[s]: the coder of segment s.  As in plan_batch, the bool-coded segments come first in the batch's records
// (BatchPlan::seg_out) and in the launch order; an rANS-coded segment's stream lands in its token slot, not in caps[s].
int lepb200_encode_upload_tokens_coded(lepb200_ctx* ctx, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* caps, int nseg,
                                       const int32_t* seg_per_file, int nfiles, const uint8_t* coders) {
    if (!ctx || !tokens || !ntok || !caps || nseg <= 0 || !seg_per_file || nfiles <= 0) return LEPB200_ERR_INVALID;
    for (int s = 0; coders && s < nseg; ++s)
        if (coders[s] > LEPB200_CODER_ANS) { ctx->err = "encode_upload_tokens: invalid entropy coder"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    ctx->have_batch = ctx->launched = ctx->symbolised = ctx->decode_fetched = false; ctx->is_encode = true; ctx->canary = true;
    BatchPlan& b = ctx->batch;
    b.images.assign(nfiles, ImageDesc());
    b.segs.assign(nseg, SegDesc());
    b.seg_blocks.assign(nseg, 0);
    b.plane_bytes.assign((size_t)nfiles * 3, 0);
    b.plane_total = b.stream_total = b.row_stride = 0;
    b.tokens_known = true;
    b.token_total = 0;
    int s = 0;
    for (int f = 0; f < nfiles; ++f) {
        if (seg_per_file[f] < 1 || seg_per_file[f] > nseg - s) { ctx->err = "encode_upload_tokens: seg_per_file does not add up to nseg"; return LEPB200_ERR_INVALID; }
        for (int k = 0; k < seg_per_file[f]; ++k, ++s) {
            SegDesc& sd = b.segs[s];
            sd.image = f;
            sd.is_last = k + 1 == seg_per_file[f];
            sd.ntok = ntok[s];
            sd.tok_cap = token_slot(ntok[s]);
            if (sd.ntok > sd.tok_cap) { ctx->err = "encode_upload_tokens: token stream too long"; return LEPB200_ERR_INVALID; }
            sd.tokens = b.token_total;
            b.token_total += sd.tok_cap;
            sd.stream = b.stream_total;
            sd.cap = caps[s];
            b.stream_total += align_up((size_t)caps[s] + CANARY_BYTES, 256);
        }
    }
    if (s != nseg) { ctx->err = "encode_upload_tokens: seg_per_file does not add up to nseg"; return LEPB200_ERR_INVALID; }
    std::vector<uint16_t> tok((size_t)b.token_total, 0);
    size_t src = 0;
    for (int i = 0; i < nseg; ++i) { memcpy(tok.data() + b.segs[i].tokens, tokens + src, (size_t)ntok[i] * 2); src += ntok[i]; }
    auto ans = [&](int x) { return coders && coders[x] == LEPB200_CODER_ANS; };
    b.seg_out.clear();
    if (coders && std::any_of(coders, coders + nseg, [](uint8_t c) { return c == LEPB200_CODER_ANS; })) {
        b.seg_out.resize(nseg);
        for (int i = 0; i < nseg; ++i) b.seg_out[i] = i;
        std::stable_partition(b.seg_out.begin(), b.seg_out.end(), [&](int x) { return !ans(x); });
        std::vector<SegDesc> segs(nseg);
        for (int d = 0; d < nseg; ++d) segs[d] = b.segs[b.seg_out[d]];
        b.segs.swap(segs);
    }
    auto caller = [&](int d) { return b.seg_out.empty() ? d : b.seg_out[d]; };
    b.order.resize(nseg);
    for (int i = 0; i < nseg; ++i) b.order[i] = i;
    std::stable_sort(b.order.begin(), b.order.end(), [&](int x, int y) {
        return ans(caller(x)) != ans(caller(y)) ? ans(caller(y)) : ntok[caller(x)] > ntok[caller(y)]; });
    b.order_ans = nseg;
    while (b.order_ans > 0 && ans(caller(b.order[b.order_ans - 1]))) --b.order_ans;
    CK(ctx->d_streams.reserve(b.stream_total + 256));
    CK(ctx->d_tokens.reserve((size_t)b.token_total * 2 + 256));
    CK(ctx->d_images.reserve(sizeof(ImageDesc) * nfiles));
    CK(ctx->d_segs.reserve(sizeof(SegDesc) * nseg));
    CK(ctx->d_order.reserve(sizeof(int) * nseg));
    CK(ctx->d_counter.reserve(256));
    for (auto& sd : b.segs) sd.stream += (unsigned long long)(uintptr_t)ctx->d_streams.p;
    CK(cudaMemsetAsync(ctx->d_streams.p, CANARY_BYTE, b.stream_total, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_tokens.p, tok.data(), tok.size() * 2, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_images.p, b.images.data(), sizeof(ImageDesc) * nfiles, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_segs.p, b.segs.data(), sizeof(SegDesc) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaMemcpyAsync(ctx->d_order.p, b.order.data(), sizeof(int) * nseg, cudaMemcpyHostToDevice, ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    CK(cudaEventRecord(ctx->ev_mid, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    ctx->have_batch = ctx->symbolised = true;
    return LEPB200_OK;
}

// After lepb200_encode_fetch(_files) of a lepb200_encode_upload_tokens batch: moved[s] = 1 where stream s ended up in the
// overflow arena, *changed = canary bytes that are no longer canary bytes, behind every slot and behind the overflow arena.
int lepb200_encode_token_canaries(lepb200_ctx* ctx, uint8_t* moved, uint64_t* changed) {
    if (!ctx || !moved || !changed || !ctx->canary || !ctx->launched) { if (ctx) ctx->err = "encode_token_canaries without a fetched token batch"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const BatchPlan& b = ctx->batch;
    const int nseg = (int)b.segs.size();
    std::vector<SegDesc> hs(nseg);
    std::vector<uint8_t> arena(b.stream_total), tail(ctx->rc_ovf_used ? CANARY_BYTES : 0);
    CK(cudaMemcpyAsync(hs.data(), ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(arena.data(), ctx->d_streams.p, b.stream_total, cudaMemcpyDeviceToHost, ctx->stream));
    if (!tail.empty()) CK(cudaMemcpyAsync(tail.data(), static_cast<uint8_t*>(ctx->d_rc_ovf.p) + ctx->rc_ovf_used, CANARY_BYTES, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    const unsigned long long base = (unsigned long long)(uintptr_t)ctx->d_streams.p;
    uint64_t bad = 0;
    for (int s = 0; s < nseg; ++s) {
        const size_t slot = (size_t)(b.segs[s].stream - base), end = slot + align_up((size_t)b.segs[s].cap + CANARY_BYTES, 256);
        for (size_t k = slot + b.segs[s].cap; k < end; ++k) bad += arena[k] != CANARY_BYTE;
        moved[b.seg_out.empty() ? s : b.seg_out[s]] = hs[s].stream < base || hs[s].stream >= base + b.stream_total;
    }
    for (uint8_t c : tail) bad += c != CANARY_BYTE;
    *changed = bad;
    return LEPB200_OK;
}

// ------------------------------------------------------------------------------------------------ GPU Huffman encode
static int henc_launch(lepb200_ctx* ctx, lepb200_henc_image* imgs, int n, int nparts) {
    if (!ctx || !imgs || n <= 0) return LEPB200_ERR_INVALID;
    ctx->henc_parts.clear();
    if (!ctx->launched || ctx->is_encode || n != (int)ctx->batch.images.size()) { ctx->err = "huffman_encode_resident: needs the decode batch just launched on this context"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    HuffEncodePlan& p = ctx->henc;
    plan_huffman_encode(p, imgs, n, ctx->batch.images.data());
    std::vector<HEncImage>& hi = p.images;
    const std::vector<HEncSeg>& hs = p.segs;
    const std::vector<HEncTable>& tabs = p.tabs.tabs;
    const size_t total = p.total;
    if (hs.empty()) return LEPB200_OK;
    CK(ctx->d_henc_out.reserve(total + 256));
    CK(ctx->d_henc_imgs.reserve(sizeof(HEncImage) * n));
    CK(ctx->d_henc_segs.reserve(sizeof(HEncSeg) * hs.size()));
    CK(ctx->d_henc_tabs.reserve(sizeof(HEncTable) * std::max<size_t>(1, tabs.size())));
    for (int i = 0; i < n; ++i) if (p.off[i] != SIZE_MAX) hi[i].out += (unsigned long long)(uintptr_t)ctx->d_henc_out.p;
    // the records travel from pinned memory: a copy from pageable memory of this size would hold the calling thread
    // until the stream has reached it, i.e. for the whole decode kernel queued in front
    {
        const size_t b_img = align_up(sizeof(HEncImage) * (size_t)n, 256), b_seg = align_up(sizeof(HEncSeg) * hs.size(), 256), b_tab = sizeof(HEncTable) * tabs.size();
        CK(ctx->h_henc_desc.reserve(b_img + b_seg + b_tab + 256));
        uint8_t* hd = static_cast<uint8_t*>(ctx->h_henc_desc.p);
        memcpy(hd, hi.data(), sizeof(HEncImage) * (size_t)n);
        memcpy(hd + b_img, hs.data(), sizeof(HEncSeg) * hs.size());
        memcpy(hd + b_img + b_seg, tabs.data(), b_tab);
        CK(cudaMemcpyAsync(ctx->d_henc_imgs.p, hd, sizeof(HEncImage) * n, cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_henc_segs.p, hd + b_img, sizeof(HEncSeg) * hs.size(), cudaMemcpyHostToDevice, ctx->stream));
        CK(cudaMemcpyAsync(ctx->d_henc_tabs.p, hd + b_img + b_seg, b_tab, cudaMemcpyHostToDevice, ctx->stream));
    }
    const int nseg = (int)hs.size();
    if (nparts <= 0) {                    // one launch, the caller fetches everything with lepb200_huffman_encode_fetch
        lep_huffencode_kernel<<<(nseg + HENC_WARPS - 1) / HENC_WARPS, HENC_WARPS * 32, 0, ctx->stream>>>(
            static_cast<const HEncImage*>(ctx->d_henc_imgs.p), static_cast<HEncSeg*>(ctx->d_henc_segs.p), nseg, static_cast<const HEncTable*>(ctx->d_henc_tabs.p));
        CK(cudaGetLastError());
        ctx->launches += 1;
        return LEPB200_OK;
    }
    // parts of consecutive images with about equal output bytes: one launch each, and behind each launch the D2H of its
    // scan bytes and segment records on the copy stream -- part k travels (and the host assembles its files) while
    // part k + 1 is encoded
    CK(ctx->h_henc_out.reserve(total + 256));
    CK(ctx->h_henc_segs.reserve(sizeof(HEncSeg) * hs.size()));
    while (ctx->part_events.size() < 2 * (size_t)nparts) {
        cudaEvent_t e;
        CK(cudaEventCreateWithFlags(&e, cudaEventDisableTiming));
        ctx->part_events.push_back(e);
    }
    // the decode batch's segment records first: they must not queue behind the part copies on the copy stream
    {
        const int nseg_dec = (int)ctx->batch.segs.size();
        CK(ctx->h_segs.reserve(sizeof(SegDesc) * nseg_dec));
        if (!ctx->status_ev) CK(cudaEventCreateWithFlags(&ctx->status_ev, cudaEventDisableTiming));
        CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev1, 0));
        CK(cudaMemcpyAsync(ctx->h_segs.p, ctx->d_segs.p, sizeof(SegDesc) * nseg_dec, cudaMemcpyDeviceToHost, ctx->copy_stream));
        CK(cudaEventRecord(ctx->status_ev, ctx->copy_stream));
        ctx->status_queued = true;
    }
    int i0 = 0;
    for (int k = 0; k < nparts && i0 < n; ++k) {
        const size_t want_end = k + 1 == nparts ? total : total / nparts * (k + 1);
        int i1 = i0;
        size_t bend = 0;
        auto end_of = [&](int i) { return p.off[i] == SIZE_MAX ? (size_t)0 : p.off[i] + align_up((size_t)imgs[i].scan_bytes + 16, 256); };
        while (i1 < n && (k + 1 == nparts || std::max(bend, end_of(i1)) <= want_end || i1 == i0)) { bend = std::max(bend, end_of(i1)); ++i1; }
        lepb200_ctx::HEncPart pt;
        pt.i0 = i0; pt.i1 = i1; pt.s0 = -1; pt.s1 = -1; pt.b0 = SIZE_MAX; pt.b1 = 0; pt.done = ctx->part_events[2 * k + 1];
        for (int i = i0; i < i1; ++i) {
            if (p.off[i] == SIZE_MAX) continue;
            if (pt.s0 < 0) pt.s0 = p.seg_first[i];
            pt.s1 = p.seg_first[i] + imgs[i].nseg;
            pt.b0 = std::min(pt.b0, p.off[i]);
            pt.b1 = std::max(pt.b1, p.off[i] + (size_t)imgs[i].scan_bytes);
        }
        if (pt.s0 >= 0) {
            const int ns = pt.s1 - pt.s0;
            lep_huffencode_kernel<<<(ns + HENC_WARPS - 1) / HENC_WARPS, HENC_WARPS * 32, 0, ctx->stream>>>(
                static_cast<const HEncImage*>(ctx->d_henc_imgs.p), static_cast<HEncSeg*>(ctx->d_henc_segs.p) + pt.s0, ns, static_cast<const HEncTable*>(ctx->d_henc_tabs.p));
            CK(cudaGetLastError());
            ctx->launches += 1;
            CK(cudaEventRecord(ctx->part_events[2 * k], ctx->stream));
            CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->part_events[2 * k], 0));
            CK(cudaMemcpyAsync(static_cast<uint8_t*>(ctx->h_henc_out.p) + pt.b0, static_cast<const uint8_t*>(ctx->d_henc_out.p) + pt.b0, pt.b1 - pt.b0, cudaMemcpyDeviceToHost, ctx->copy_stream));
            CK(cudaMemcpyAsync(static_cast<HEncSeg*>(ctx->h_henc_segs.p) + pt.s0, static_cast<const HEncSeg*>(ctx->d_henc_segs.p) + pt.s0, sizeof(HEncSeg) * (size_t)ns, cudaMemcpyDeviceToHost, ctx->copy_stream));
        }
        CK(cudaEventRecord(pt.done, ctx->copy_stream));
        ctx->henc_parts.push_back(pt);
        i0 = i1;
    }
    return LEPB200_OK;
}

int lepb200_huffman_encode_resident(lepb200_ctx* ctx, lepb200_henc_image* imgs, int n) { return henc_launch(ctx, imgs, n, 0); }

int lepb200_huffman_encode_resident_parts(lepb200_ctx* ctx, lepb200_henc_image* imgs, int n, int nparts) {
    return henc_launch(ctx, imgs, n, std::max(1, std::min(16, nparts)));
}

int lepb200_huffman_encode_parts(const lepb200_ctx* ctx) { return ctx ? (int)ctx->henc_parts.size() : 0; }

// data / status of images [i0, i1) from the fetched scan bytes and segment records
static void henc_results(const lepb200_ctx* ctx, lepb200_henc_image* imgs, int i0, int i1) {
    const HuffEncodePlan& p = ctx->henc;
    const HEncSeg* hs = static_cast<const HEncSeg*>(ctx->h_henc_segs.p);
    for (int i = i0; i < i1; ++i) {
        if (p.off[i] == SIZE_MAX) continue;
        imgs[i].data = static_cast<const uint8_t*>(ctx->h_henc_out.p) + p.off[i];
        int st = 0;
        for (int k = 0; k < p.seg_count[i]; ++k) if (hs[p.seg_first[i] + k].status) st = 1;
        imgs[i].status = st;
    }
}

int lepb200_huffman_encode_wait_part(lepb200_ctx* ctx, lepb200_henc_image* imgs, int n, int part, int* first, int* last) {
    if (!ctx || !imgs || !first || !last || n != (int)ctx->henc.off.size() || part < 0 || part >= (int)ctx->henc_parts.size()) return LEPB200_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    const lepb200_ctx::HEncPart& pt = ctx->henc_parts[part];
    CK(cudaEventSynchronize(pt.done));
    henc_results(ctx, imgs, pt.i0, pt.i1);
    *first = pt.i0; *last = pt.i1;
    return LEPB200_OK;
}

int lepb200_huffman_encode_fetch(lepb200_ctx* ctx, lepb200_henc_image* imgs, int n) {
    if (!ctx || !imgs || n != (int)ctx->henc.off.size()) return LEPB200_ERR_INVALID;
    const HuffEncodePlan& p = ctx->henc;
    if (p.segs.empty()) return LEPB200_OK;
    CK(cudaSetDevice(ctx->device));
    size_t total = 0;
    for (int i = 0; i < n; ++i) if (p.off[i] != SIZE_MAX) total = std::max(total, p.off[i] + imgs[i].scan_bytes);
    CK(ctx->h_henc_out.reserve(total + 256));
    CK(ctx->h_henc_segs.reserve(sizeof(HEncSeg) * p.segs.size()));
    CK(cudaMemcpyAsync(ctx->h_henc_out.p, ctx->d_henc_out.p, total, cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaMemcpyAsync(ctx->h_henc_segs.p, ctx->d_henc_segs.p, sizeof(HEncSeg) * p.segs.size(), cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    henc_results(ctx, imgs, 0, n);
    return LEPB200_OK;
}

int lepb200_huffman_encode_adler32(lepb200_ctx* ctx, int first, int last, uint32_t* adler) {
    if (!ctx || !adler || first < 0 || first > last || last > (int)ctx->henc.off.size()) return LEPB200_ERR_INVALID;
    const HuffEncodePlan& p = ctx->henc;
    const HEncSeg* hs = static_cast<const HEncSeg*>(ctx->h_henc_segs.p);
    for (int i = first; i < last; ++i) {
        uLong a = adler32(0L, Z_NULL, 0);
        for (int k = 0; p.off[i] != SIZE_MAX && k < p.seg_count[i]; ++k) {     // segments lie back to back, in order
            const HEncSeg& sg = hs[p.seg_first[i] + k];
            a = adler32_combine(a, sg.adler, (z_off_t)sg.produced);
        }
        adler[i] = (uint32_t)a;
    }
    return LEPB200_OK;
}

// ------------------------------------------------------------------------------------------------ decode
static int decode_upload_impl(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                              const lepb200_buffer* spans, const uint32_t* span_first, const uint8_t* coders) {
    if (!ctx || !in) return LEPB200_ERR_INVALID;
    CK(cudaSetDevice(ctx->device));
    ctx->d_tokens.release();              // the encoder's token arena (the largest buffer of that direction) is not needed on the way back
    int r = build_batch(ctx, images, nimages, false, in, coders);
    if (r) return r;
    const int nseg = (int)ctx->batch.segs.size();
    // planes start zeroed: blocks outside the coded range (truncated images) stay zero like the reference's calloc.
    // Issued first: the device clears them while the host packs the streams.
    CK(cudaMemsetAsync(ctx->d_planes.p, 0, ctx->batch.plane_total, ctx->stream));
    // pack the streams into the pinned staging buffer (over a gigabyte for a 4096-image batch: a single-threaded copy
    // loop took longer than the H2D itself) in a few slices of consecutive segments; every slice is packed by the
    // context's host threads and its H2D copy runs while the next one is packed
    const unsigned long long base = (unsigned long long)(uintptr_t)ctx->d_streams.p;
    size_t total = 0;
    for (int s = 0; s < nseg; ++s) total = std::max(total, (size_t)(ctx->batch.segs[s].stream - base) + in[s].len);
    CK(ctx->h_stage.reserve(total + 16));
    uint8_t* hs = static_cast<uint8_t*>(ctx->h_stage.p);
    const int nslices = total > (size_t(64) << 20) ? 8 : 1;
    int s0 = 0;
    for (int k = 0; k < nslices && s0 < nseg; ++k) {
        // segments are laid out in order, so a slice is a contiguous byte range of the staging buffer
        const size_t want_end = total / nslices * (k + 1);
        int s1 = s0;
        while (s1 < nseg && (k + 1 == nslices || (size_t)(ctx->batch.segs[s1].stream - base) < want_end)) ++s1;
        const int nt = std::max(1, std::min(ctx->host_threads, s1 - s0));
        auto pack = [&](int t) {
            for (int s = s0 + t; s < s1; s += nt) {
                uint8_t* dst = hs + (ctx->batch.segs[s].stream - base);
                if (!spans) { if (in[s].len) memcpy(dst, in[s].data, in[s].len); continue; }
                size_t room = in[s].len;                       // the pieces of a stream as they lie in the caller's file
                for (uint32_t q = span_first[s]; q < span_first[s + 1] && room; ++q) {
                    const size_t n = std::min(room, spans[q].len);
                    memcpy(dst, spans[q].data, n);
                    dst += n; room -= n;
                }
            }
        };
        if (nt == 1) pack(0);
        else {
            std::vector<std::thread> th;
            for (int t = 0; t < nt; ++t) th.emplace_back(pack, t);
            for (auto& t : th) t.join();
        }
        const size_t b0 = (size_t)(ctx->batch.segs[s0].stream - base);
        const size_t b1 = s1 < nseg ? (size_t)(ctx->batch.segs[s1].stream - base) : total;
        if (b1 > b0) CK(cudaMemcpyAsync(static_cast<uint8_t*>(ctx->d_streams.p) + b0, hs + b0, b1 - b0, cudaMemcpyHostToDevice, ctx->stream));
        s0 = s1;
    }
    ctx->have_batch = true;
    return LEPB200_OK;
}

int lepb200_decode_upload(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in) {
    return decode_upload_impl(ctx, images, nimages, in, nullptr, nullptr, nullptr);
}

int lepb200_decode_upload_gather(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                 const lepb200_buffer* spans, const uint32_t* span_first) {
    if (!spans || !span_first) return LEPB200_ERR_INVALID;
    return decode_upload_impl(ctx, images, nimages, in, spans, span_first, nullptr);
}

int lepb200_decode_upload_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                const uint8_t* coders) {
    return decode_upload_impl(ctx, images, nimages, in, nullptr, nullptr, coders);
}

int lepb200_decode_upload_gather_coded(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                       const lepb200_buffer* spans, const uint32_t* span_first, const uint8_t* coders) {
    if (!spans || !span_first) return LEPB200_ERR_INVALID;
    return decode_upload_impl(ctx, images, nimages, in, spans, span_first, coders);
}

int lepb200_decode_launch(lepb200_ctx* ctx) {
    if (!ctx || !ctx->have_batch || ctx->is_encode) { if (ctx) ctx->err = "decode_launch without decode_upload"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size();
    const int nbool = ctx->batch.order_ans;
    ctx->decode_fetched = false;
    CK(cudaMemsetAsync(ctx->d_counter.p, 0, sizeof(int), ctx->stream));
    CK(cudaEventRecord(ctx->ev0, ctx->stream));
    int r = nbool > 0 ? decode_launch_part<BoolReader, G2Bool>(ctx, 0, nbool, ctx->dec_threads, ctx->dec_group_grid, ctx->grid) : LEPB200_OK;
    if (r == LEPB200_OK && nseg > nbool)
        r = decode_launch_part<AnsReader, G2Ans>(ctx, nbool, nseg - nbool, ctx->dec_threads_ans, ctx->dec_group_grid_ans, ctx->grid_ans);
    if (r) return r;
    CK(cudaEventRecord(ctx->ev1, ctx->stream));
    ctx->status_queued = false;
    ctx->launched = true;
    return LEPB200_OK;
}

int lepb200_decode_fetch(lepb200_ctx* ctx, const lepb200_image* images, int nimages, int32_t* status_out) {
    if (!ctx || !ctx->launched || ctx->is_encode) { if (ctx) ctx->err = "decode_fetch without decode_launch"; return LEPB200_ERR_INVALID; }
    if (nimages != (int)ctx->batch.images.size()) { ctx->err = "decode_fetch: batch size mismatch"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size();
    CK(ctx->h_segs.reserve(sizeof(SegDesc) * nseg));
    SegDesc* hs = static_cast<SegDesc*>(ctx->h_segs.p);
    CK(cudaMemcpyAsync(hs, ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->stream));
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c)
            if (images[i].planes[c])        // NULL: the caller does not need this plane on the host (scan re-encoded on the device)
                CK(cudaMemcpyAsync(images[i].planes[c], reinterpret_cast<const void*>(ctx->batch.images[i].plane[c]), ctx->batch.plane_bytes[(size_t)i * 3 + c],
                                   cudaMemcpyDeviceToHost, ctx->stream));
    CK(cudaStreamSynchronize(ctx->stream));
    CK(cudaEventElapsedTime(&ctx->last_ms, ctx->ev0, ctx->ev1));
    uint64_t alg = 0;
    for (int s = 0; s < nseg; ++s) {
        if (status_out) status_out[s] = hs[s].status;
        alg += (uint64_t)ctx->batch.seg_blocks[s] * 128 + ctx->batch.segs[s].cap;
    }
    ctx->alg_bytes = alg;
    ctx->decode_fetched = true;
    return LEPB200_OK;
}

int lepb200_decode_fetch_decisions(lepb200_ctx* ctx, uint64_t* out) {
    if (!ctx || !out || !ctx->decode_fetched) { if (ctx) ctx->err = "decode_fetch_decisions without decode_fetch"; return LEPB200_ERR_INVALID; }
    const SegDesc* hs = static_cast<const SegDesc*>(ctx->h_segs.p);
    for (size_t s = 0; s < ctx->batch.segs.size(); ++s) out[s] = (uint64_t)hs[s].ndecisions_lo | ((uint64_t)hs[s].ndecisions_hi << 32);
    return LEPB200_OK;
}

int lepb200_decode_fetch_status(lepb200_ctx* ctx, int32_t* status_out) {
    if (!ctx || !status_out || !ctx->launched || ctx->is_encode) { if (ctx) ctx->err = "decode_fetch_status without decode_launch"; return LEPB200_ERR_INVALID; }
    CK(cudaSetDevice(ctx->device));
    const int nseg = (int)ctx->batch.segs.size();
    CK(ctx->h_segs.reserve(sizeof(SegDesc) * nseg));
    SegDesc* hs = static_cast<SegDesc*>(ctx->h_segs.p);
    if (ctx->status_queued) {                                            // queued by lepb200_huffman_encode_resident_parts ahead of its copies
        CK(cudaEventSynchronize(ctx->status_ev));
    } else {
        CK(cudaStreamWaitEvent(ctx->copy_stream, ctx->ev1, 0));          // the decode kernel, not what was queued behind it
        CK(cudaMemcpyAsync(hs, ctx->d_segs.p, sizeof(SegDesc) * nseg, cudaMemcpyDeviceToHost, ctx->copy_stream));
        CK(cudaStreamSynchronize(ctx->copy_stream));
    }
    for (int s = 0; s < nseg; ++s) status_out[s] = hs[s].status;
    return LEPB200_OK;
}

int lepb200_decode_images(lepb200_ctx* ctx, const lepb200_image* images, int nimages, const lepb200_stream* in, int32_t* status_out) {
    int r = lepb200_decode_upload(ctx, images, nimages, in);
    if (r) return r;
    r = lepb200_decode_launch(ctx);
    if (r) return r;
    return lepb200_decode_fetch(ctx, images, nimages, status_out);
}

}  // extern "C"
