// emu_kernels.cc -- runs the coder kernels on the CPU under the warp emulator of cuda_shim.h (test infrastructure).
//
// The kernel sources are compiled as host C++, and the job descriptors come from the same planner as the library's
// (lep_plan.cuh: ImageDesc / SegDesc, HuffJob, HEncImage / HEncSeg, arena offsets, launch order).  This file rebases the
// planned offsets onto host vectors (poisoned where the device arena is not cleared), launches the kernels with their
// device launch shapes and runs the host steps between launches.  Entry points mirror the C ABI (include/lepton_b200.h).
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "cuda_shim.h"
#include "../../lepton_b200/csrc/lep_encode.cu"
#include "../../lepton_b200/csrc/lep_decode.cu"
#include "../../lepton_b200/csrc/lep_decode_g2.cu"
#include "../../lepton_b200/csrc/lep_huffpar.cu"
#include "../../lepton_b200/csrc/lep_mux.cu"
#include "../../lepton_b200/csrc/lep_huffenc.cu"
#include "../../lepton_b200/csrc/lep_plan.cuh"
#include "../../include/lepton_b200.h"

using namespace lepb200;

namespace {

// host arena: a vector of n bytes + 512 filled with `fill`, used from its first 256-byte aligned byte (like a device allocation)
uint8_t* host_arena(std::vector<uint8_t>& v, size_t n, uint8_t fill) {
    v.assign(n + 512, fill);
    return reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)v.data(), 256));
}

// plane and stream offsets of a batch plan -> addresses in the host arenas
void rebase(BatchPlan& b, uint8_t* planes, uint8_t* streams) {
    for (auto& d : b.images)
        for (int c = 0; c < d.ncmp; ++c) d.plane[c] += (unsigned long long)(uintptr_t)planes;
    for (auto& sd : b.segs) sd.stream += (unsigned long long)(uintptr_t)streams;
}

struct LaunchArgs {
    int kernel;
    const ImageDesc* images; SegDesc* segs; int nseg; const int* order; int* counter;
    uint16_t* models; uint8_t* rows; size_t row_stride;
};

void kernel_body(void* p) {
    const LaunchArgs& a = *static_cast<const LaunchArgs*>(p);
    if (a.kernel == 0) lep_decode_kernel(a.images, a.segs, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 201) lep_decode_g2_kernel<1>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 202) lep_decode_g2_kernel<2>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 204) lep_decode_g2_kernel<4>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 208) lep_decode_g2_kernel<8>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 216) lep_decode_g2_kernel<16>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else lep_decode_g2_kernel<32>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
}

// launch shape of the group kernel: warps per CTA and thread-segments per warp for G lanes per segment
void group_shape(int G, int& warps, int& per_warp) {
    per_warp = 32 / G;
    warps = G >= 4 ? 4 : G;
}

}  // namespace

// kernel: 0 = lep_decode_kernel (warp per segment, persistent CTAs; `grid_cap` > 0 limits the CTAs so that warps take
// several segments from the queue), 200 + G = lep_decode_g2_kernel<G> (G lanes per segment).  Decodes into images[i].planes (zeroed first,
// like the device arena); per-segment status and decision counts come back like lepb200_decode_fetch reports them.
// reverse = 1 runs the launch's CTAs and threads in reverse order (emu::g_reverse).
extern "C" int emu_decode_images(int kernel, int grid_cap, int reverse, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                 int32_t* status_out, uint64_t* ndecisions_out) {
    const int gl = kernel % 100;
    const bool group = kernel / 100 == 2 && (gl == 1 || gl == 2 || gl == 4 || gl == 8 || gl == 16 || gl == 32);
    if (!in || (kernel != 0 && !group)) return LEPB200_ERR_INVALID;
    BatchPlan b;
    if (plan_batch(b, images, nimages, false, in)) return LEPB200_ERR_INVALID;
    const int nseg = (int)b.segs.size();
    // planes start zeroed like the device arena; the stream arena is not cleared: whatever is behind a stream must not matter
    std::vector<uint8_t> pv, sv;
    uint8_t* pbase = host_arena(pv, b.plane_total, 0);
    uint8_t* sbase = host_arena(sv, b.stream_total, 0xA5);
    for (int s = 0; s < nseg; ++s) if (in[s].len) memcpy(sbase + b.segs[s].stream, in[s].data, (size_t)in[s].len);
    rebase(b, pbase, sbase);
    std::vector<SegDesc>& segs = b.segs;
    LaunchArgs a;
    a.kernel = kernel; a.images = b.images.data(); a.segs = segs.data(); a.nseg = nseg; a.order = b.order.data(); a.row_stride = b.row_stride;
    int counter = 0;
    a.counter = &counter;
    unsigned grid, block;
    size_t group_slots = 0;
    if (group) {
        // 100 + G: lep_decode_group_kernel<G>; grid_cap > 0 limits the CTAs so that groups take several segments from the queue
        int warps, per_warp;
        group_shape(kernel % 100, warps, per_warp);
        grid = (unsigned)((nseg + warps * per_warp - 1) / (warps * per_warp));
        if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
        block = (unsigned)warps * 32;
        group_slots = (size_t)grid * warps * per_warp;
    } else {
        grid = (unsigned)((nseg + DEC_WARPS_PER_CTA - 1) / DEC_WARPS_PER_CTA);
        if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
        block = DEC_WARPS_PER_CTA * 32;
    }
    const size_t slots = kernel == 0 ? (size_t)grid * DEC_WARPS_PER_CTA : (size_t)nseg;
    std::vector<uint16_t> models(slots * M_TOTAL, kernel == 0 ? 0x5a5a : 0);       // thread / group kernels: zero fill before the launch; the warp kernel clears its own
    std::vector<uint8_t> rows((group ? group_slots : slots) * b.row_stride, 0);
    a.models = models.data(); a.rows = rows.data();
    emu::g_reverse = reverse != 0;
    emu::launch(grid, block, kernel_body, &a);
    emu::g_reverse = false;
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c)
            memcpy(images[i].planes[c], reinterpret_cast<const void*>(b.images[i].plane[c]), b.plane_bytes[(size_t)i * 3 + c]);
    for (int s = 0; s < nseg; ++s) {
        if (status_out) status_out[s] = segs[s].status;
        if (ndecisions_out) ndecisions_out[s] = (uint64_t)segs[s].ndecisions_lo | ((uint64_t)segs[s].ndecisions_hi << 32);
    }
    return 0;
}

namespace {

struct EncArgs {
    int stage;                       // 0 count, 1 offsets, 2 symbolise (kernel A), 3 range coder (kernel B)
    const ImageDesc* images; SegDesc* segs; int nseg; const int* order; int* counter;
    uint16_t* models; uint8_t* rows; size_t row_stride; uint16_t* tokens; unsigned long long* total;
    unsigned long long* ck; uint32_t* digits; uint8_t* ovf;
};

void enc_body(void* p) {
    const EncArgs& a = *static_cast<const EncArgs*>(p);
    if (a.stage == 0) lep_count_kernel(a.images, a.segs, a.nseg);
    else if (a.stage == 1) lep_token_offsets_kernel(a.segs, a.nseg, a.total);
    else if (a.stage == 2) lep_encode_kernel(a.images, a.segs, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride, a.tokens);
    else if (a.stage == 3) lep_rangecode_kernel(a.segs, a.nseg, a.order, a.tokens);
    else if (a.stage == 5) lep_rangepass_kernel<true>(a.segs, a.nseg, a.order, a.tokens, a.ck);
    else if (a.stage == 4) lep_rangepass_kernel<false>(a.segs, a.nseg, a.order, a.tokens, a.ck);
    else if (a.stage == 6) lep_digit_offsets_kernel(a.segs, a.nseg, a.total, a.total + 1);
    else if (a.stage == 7) lep_rangepiece_kernel(a.segs, a.nseg, a.tokens, a.ck, a.digits);
    else lep_rangenorm_kernel(a.segs, a.nseg, a.order, a.digits, a.ovf);
}

// Kernel B after kernel A, with the launch shapes and the host steps of lepb200_encode_launch_rangecode /
// lepb200_encode_fetch (lep_capi.cu): kernel 0 / 2 = the parallel range coder (async / register token feed): range pass,
// digit offsets (+ overflow slots: `ovf` receives the overflow arena), pieces, carries; kernel 1 = the serial coder, then
// plan_serial_rerun for the segments whose stream outgrew the slot.  `total_tokens` = size of the token arena.
void run_range_coder(int kernel, EncArgs& a, unsigned long long total_tokens, std::vector<uint8_t>& ovf) {
    const int nseg = a.nseg;
    std::vector<unsigned long long> ck;
    std::vector<uint32_t> digits;
    if (kernel == 0 || kernel == 2) {
        ck.assign(rc_checkpoints(total_tokens, nseg), 0);
        a.ck = ck.data();
        a.stage = kernel == 0 ? 5 : 4; emu::launch((unsigned)((nseg + RCT_THREADS - 1) / RCT_THREADS), RCT_THREADS, enc_body, &a);
        unsigned long long totals[2] = {0, 0};
        a.total = totals;
        a.stage = 6; emu::launch(1, 1024, enc_body, &a);
        digits.assign((size_t)totals[0] + 64, 0);
        ovf.assign((size_t)totals[1] + 256, 0xC3);                 // + 256 canary bytes (emu_range_code)
        a.digits = digits.data();
        a.ovf = ovf.data();
        a.stage = 7;
        for (int y = 0; y < nseg; ++y) { emu::g_block_idx.y = (unsigned)y; emu::launch(8, RCP_THREADS, enc_body, &a); }      // grid (8, nseg)
        emu::g_block_idx.y = 0;
        a.stage = 8; emu::launch((unsigned)((nseg + RCN_WARPS - 1) / RCN_WARPS), RCN_WARPS * 32, enc_body, &a);
        return;
    }
    a.stage = 3; emu::launch((unsigned)((nseg + RC_THREADS - 1) / RC_THREADS), RC_THREADS, enc_body, &a);
    std::vector<int> redo;
    const size_t total = plan_serial_rerun(a.segs, nseg, redo);
    if (redo.empty()) return;
    ovf.assign(total + 256, 0xC3);
    for (int s : redo) a.segs[s].stream += (unsigned long long)(uintptr_t)ovf.data();
    const int* order = a.order;
    a.order = redo.data(); a.nseg = (int)redo.size();
    a.stage = 3; emu::launch((unsigned)((redo.size() + RC_THREADS - 1) / RC_THREADS), RC_THREADS, enc_body, &a);
    a.order = order; a.nseg = nseg;
}

}  // namespace

// lepb200_encode_images on the emulator: count pre-pass -> token offsets -> kernel A (symbolise + model) -> kernel B
// (range coder), with the launch shapes of lep_capi.cu.  `out` must hold sum(nseg) entries; the bytes of every stream are
// copied into `arena` (capacity arena_cap) back to back and out[i].data points there.  grid_cap > 0 limits kernel A's
// CTAs (persistent warps then take several segments each).  kernel: 0 = parallel range coder, 1 = serial range coder,
// 2 = parallel range coder whose range pass feeds tokens through registers (LEPB200_RC_FEED=0).  tok_caps (optional,
// sum(nseg) entries) receives the token bound of every segment (the count pre-pass's, or the caller's seg_token_bound).
// reverse = 1 runs the CTAs and threads of every launch in reverse order (emu::g_reverse).
extern "C" int emu_encode_images(int kernel, int grid_cap, int reverse, const lepb200_image* images, int nimages, lepb200_stream* out, uint8_t* arena,
                                 size_t arena_cap, uint32_t* tok_caps) {
    if (!out || !arena) return LEPB200_ERR_INVALID;
    BatchPlan b;
    if (plan_batch(b, images, nimages, true, nullptr)) return LEPB200_ERR_INVALID;
    const int nseg = (int)b.segs.size();
    emu::g_reverse = reverse != 0;
    std::vector<uint8_t> pv, sv;
    uint8_t* pbase = host_arena(pv, b.plane_total, 0);
    uint8_t* sbase = host_arena(sv, b.stream_total, 0);
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c) memcpy(pbase + b.images[i].plane[c], images[i].planes[c], b.plane_bytes[(size_t)i * 3 + c]);
    rebase(b, pbase, sbase);
    std::vector<SegDesc>& segs = b.segs;

    EncArgs a;
    a.images = b.images.data(); a.segs = segs.data(); a.nseg = nseg; a.order = b.order.data(); a.row_stride = b.row_stride;
    int counter = 0;
    unsigned long long total_tokens = b.token_total;
    a.counter = &counter; a.total = &total_tokens; a.models = nullptr; a.rows = nullptr; a.tokens = nullptr;
    if (!b.tokens_known) {            // count pre-pass -> token offsets, unless every segment came with a bound
        a.stage = 0; emu::launch((unsigned)nseg, CNT_THREADS, enc_body, &a);
        a.stage = 1; emu::launch(1, 1024, enc_body, &a);
    }
    std::vector<uint16_t> tokens((size_t)total_tokens + 128, 0);
    a.tokens = tokens.data();
    std::vector<uint16_t> models;
    std::vector<uint8_t> rows;
    {
        unsigned grid = (unsigned)((nseg + ENC_WARPS_PER_CTA - 1) / ENC_WARPS_PER_CTA);
        if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
        models.assign((size_t)grid * ENC_WARPS_PER_CTA * M_TOTAL, 0x5a5a);      // the kernel clears its own
        rows.assign((size_t)grid * ENC_WARPS_PER_CTA * b.row_stride, 0);
        a.models = models.data(); a.rows = rows.data();
        a.stage = 2; emu::launch(grid, ENC_WARPS_PER_CTA * 32, enc_body, &a);
    }
    if (const char* dump = getenv("EMU_DUMP_TOKENS")) {          // diagnostics: the (probability, bit) tokens of every segment
        FILE* f = fopen(dump, "wb");
        for (int s = 0; f && s < nseg; ++s) { const uint32_t nt = segs[s].ntok; fwrite(&nt, 4, 1, f); fwrite(tokens.data() + segs[s].tokens, 2, nt, f); }
        if (f) fclose(f);
    }
    // parallel range coder (lep_capi.cu: rc_mode 1; kernel 2 = register-ring token feed) or the serial one (kernel 1, rc_mode 0)
    std::vector<uint8_t> ovf;
    run_range_coder(kernel, a, total_tokens, ovf);
    emu::g_reverse = false;
    if (tok_caps) for (int s = 0; s < nseg; ++s) tok_caps[s] = segs[s].tok_cap;
    size_t used = 0;
    for (int s = 0; s < nseg; ++s) {
        const size_t n = segs[s].status == 0 ? segs[s].len : 0;
        if (used + n > arena_cap) return LEPB200_ERR_NOMEM;
        memcpy(arena + used, reinterpret_cast<const uint8_t*>(segs[s].stream), n);
        out[s].data = arena + used;
        out[s].len = n;
        out[s].status = segs[s].status;
        out[s].reserved = 0;
        out[s].ndecisions = (uint64_t)segs[s].ndecisions_lo | ((uint64_t)segs[s].ndecisions_hi << 32);
        used += n;
    }
    return 0;
}


// ---- kernel B alone on given token streams.  Segment s has ntok[s] tokens (prob | bit << 8, all segments back to back in
// `tokens`) and a stream slot of caps[s] bytes.  The tokens are laid out like lep_token_offsets_kernel lays them out (tok_cap
// = ntok rounded up to 64 tokens after 64 of slack, so piece checkpoints sit at (tokens >> 10) + 2 * segment), the
// segments run in the order of lepb200_encode (longest first), and kernel B runs as run_range_coder runs it, overflow
// handling included.  256 canary bytes follow every slot and the overflow arena.  reverse = 1 runs every launch's
// CTAs and threads in reverse order (emu::g_reverse).  Outputs per segment: status, len, moved (1 = the stream ended up in the
// overflow arena), its bytes back to back in `out` (out_cap bytes); *canary_bad = canary bytes that changed.
extern "C" int emu_range_code(int kernel, int reverse, int nseg, const uint16_t* tokens, const uint32_t* ntok, const uint32_t* caps,
                              int32_t* status_out, uint32_t* len_out, uint8_t* moved_out, uint8_t* out, size_t out_cap, uint64_t* canary_bad) {
    if (nseg <= 0 || !tokens || !ntok || !caps || !out || !canary_bad || (kernel != 0 && kernel != 1 && kernel != 2)) return LEPB200_ERR_INVALID;
    constexpr size_t CANARY = 256;
    constexpr uint8_t CANARY_BYTE = 0xC3;
    std::vector<SegDesc> segs(nseg);
    std::vector<size_t> slot(nseg);
    unsigned long long total_tokens = 0;
    size_t stream_total = 0, src = 0;
    for (int s = 0; s < nseg; ++s) {
        SegDesc& sd = segs[s];
        memset(&sd, 0, sizeof(sd));
        sd.ntok = ntok[s];
        sd.tok_cap = token_slot(ntok[s]);
        sd.tokens = total_tokens;
        total_tokens += sd.tok_cap;
        sd.cap = caps[s];
        slot[s] = stream_total;
        stream_total += align_up((size_t)caps[s] + CANARY, 256);
    }
    std::vector<uint16_t> tok((size_t)total_tokens + 128, 0);
    for (int s = 0; s < nseg; ++s) { memcpy(tok.data() + segs[s].tokens, tokens + src, (size_t)ntok[s] * 2); src += ntok[s]; }
    std::vector<uint8_t> streams(stream_total + 256, CANARY_BYTE);
    uint8_t* sbase = reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)streams.data(), 256));
    for (int s = 0; s < nseg; ++s) segs[s].stream = (unsigned long long)(uintptr_t)(sbase + slot[s]);
    std::vector<int> order(nseg);
    for (int i = 0; i < nseg; ++i) order[i] = i;
    std::stable_sort(order.begin(), order.end(), [&](int a, int b) { return ntok[a] > ntok[b]; });
    EncArgs a;
    memset(&a, 0, sizeof(a));
    a.segs = segs.data(); a.nseg = nseg; a.order = order.data(); a.tokens = tok.data();
    std::vector<uint8_t> ovf;
    emu::g_reverse = reverse != 0;
    run_range_coder(kernel, a, total_tokens, ovf);
    emu::g_reverse = false;
    uint64_t bad = 0;
    for (int s = 0; s < nseg; ++s) {
        const uint8_t* p = sbase + slot[s];
        for (size_t k = caps[s]; k < align_up((size_t)caps[s] + CANARY, 256); ++k) bad += p[k] != CANARY_BYTE;
    }
    size_t used = 0;
    for (int s = 0; s < nseg; ++s) {
        const uint8_t* p = reinterpret_cast<const uint8_t*>(segs[s].stream);
        const bool moved = p < sbase || p >= sbase + stream_total;
        if (moved) {              // an overflow slot: the bytes of the arena behind the stream are the next slot's or the canary
            const size_t end = (size_t)(p - ovf.data()) + segs[s].cap;
            if (end > ovf.size()) return LEPB200_ERR_INVALID;
        }
        const size_t n = segs[s].status == 0 ? segs[s].len : 0;
        if (used + n > out_cap) return LEPB200_ERR_NOMEM;
        memcpy(out + used, p, n);
        used += n;
        status_out[s] = segs[s].status;
        len_out[s] = n;
        moved_out[s] = moved ? 1 : 0;
    }
    if (!ovf.empty()) for (size_t k = ovf.size() - 256; k < ovf.size(); ++k) bad += ovf[k] != CANARY_BYTE;
    *canary_bad = bad;
    return 0;
}

// ---- baseline Huffman decode: lep_huffdecode_kernel alone (mode 0) or the sub-sequence kernels of lep_huffpar.cu followed
// by it (mode 1), on the jobs of plan_huffman_decode (lep_plan.cuh), without a staging buffer.
// planes[3 * i + c] = host plane of component c of scan i (receives the decoded plane); scans[i] outputs are filled like the
// device call fills them.  info[0] = synchronisation iterations, info[1] = images the serial kernel had to redo.  reverse = 1
// runs the CTAs and threads of every launch in reverse order (emu::g_reverse).
namespace {
struct HuffArgs { HuffJob* jobs; int n; const HuffTableDev* tabs; int ntabs; HpArrays a; int iter; int last_iter; unsigned int* dirty; int which; };
void huff_body(void* p) {
    const HuffArgs& h = *static_cast<const HuffArgs*>(p);
    if (h.which == 0) lep_huffdecode_kernel(h.jobs, h.n, h.tabs, h.ntabs);
    else if (h.which == 1) lep_huffpar_sync_kernel(h.jobs, h.n, h.tabs, h.ntabs, h.a, h.iter, h.last_iter, h.dirty);
    else if (h.which == 2) lep_huffpar_prefix_kernel(h.jobs, h.n, h.a);
    else lep_huffpar_write_kernel(h.jobs, h.n, h.tabs, h.ntabs, h.a);
}
}  // namespace

extern "C" int emu_huffman_decode(int mode, int sub_bits, int iter_cap, int reverse, lepb200_jpeg_scan* scans, int n, int16_t** planes, int* info) {
    HuffDecodePlan p;
    if (plan_huffman_decode(p, scans, n, mode == 1, sub_bits, nullptr, 0)) return LEPB200_ERR_INVALID;
    emu::g_reverse = reverse != 0;
    std::vector<HuffJob>& jobs = p.jobs;
    std::vector<uint8_t> hv, rv, pv;
    uint8_t* hbase = host_arena(hv, p.huff_total, 0);              // the scans with the zero bytes the kernels read past their ends
    uint8_t* rbase = host_arena(rv, p.rows_total, 0);
    uint8_t* pbase = host_arena(pv, p.plane_total, 0);
    for (int i = 0; i < n; ++i) if (scans[i].entropy) memcpy(hbase + jobs[i].huff, scans[i].entropy, scans[i].nbytes);
    for (HuffJob& jb : jobs) {
        jb.huff += (unsigned long long)(uintptr_t)hbase;
        jb.rows += (unsigned long long)(uintptr_t)rbase;
        for (int c = 0; c < std::min(jb.ncmp, 3); ++c) jb.plane[c] += (unsigned long long)(uintptr_t)pbase;
    }
    const std::vector<HuffTableDev>& tabs = p.tabs.tabs;
    const uint32_t sub_total = p.sub_total;
    HuffArgs h;
    memset(&h, 0, sizeof(h));
    h.jobs = jobs.data(); h.n = n; h.tabs = tabs.data(); h.ntabs = (int)tabs.size();
    int iters = 0;
    std::vector<unsigned long long> ex(sub_total + 1);
    std::vector<uint32_t> epoch(sub_total + 1, 0), tok(sub_total + 1, 0);
    std::vector<uint4> cnt(sub_total + 1);
    std::vector<unsigned int> dirty(iter_cap + 4, 0);
    if (sub_total > 0) {
        h.a.exit = ex.data(); h.a.epoch = epoch.data(); h.a.cnt = cnt.data(); h.a.tok = tok.data();
        h.a.sub_base = p.sub_base.data(); h.a.total = sub_total; h.a.sub_bits = (uint32_t)sub_bits;
        h.dirty = dirty.data(); h.last_iter = iter_cap;
        const unsigned grid = (sub_total + HP_THREADS - 1) / HP_THREADS;
        h.which = 1;
        for (;;) {
            h.iter = iters;
            emu::launch(grid, HP_THREADS, huff_body, &h);
            ++iters;
            if (iters > iter_cap || dirty[iters] == 0) break;
        }
        h.which = 2; emu::launch((n + 127) / 128, 128, huff_body, &h);
        h.which = 3; emu::launch(grid, HP_THREADS, huff_body, &h);
    }
    int redo = 0;
    for (int i = 0; i < n; ++i) if (jobs[i].nsub && !(jobs[i].par_done && !jobs[i].par_redo)) ++redo;
    h.which = 0;
    emu::launch((n + 3) / 4, 4 * 32, huff_body, &h);
    emu::g_reverse = false;
    huffman_decode_results(scans, n, jobs.data(), rbase, (unsigned long long)(uintptr_t)rbase);
    for (int i = 0; i < n; ++i)
        for (int c = 0; c < std::min(jobs[i].ncmp, 3); ++c)
            if (planes[3 * i + c])
                memcpy(planes[3 * i + c], reinterpret_cast<const void*>(jobs[i].plane[c]), (size_t)jobs[i].bch[c] * jobs[i].bcv[c] * 128);
    if (info) { info[0] = iters; info[1] = redo; }
    return 0;
}


// ---- device container assembly: lep_gather_kernel over the pieces lepb200_encode_fetch_files builds (gather_file_pieces,
// lep_mux.cu) for `nfiles` files at once.  File f has header hdr[f] (hlen[f] bytes), nseg[f] streams (streams[] holds them file
// after file) and the MuxWriter plan plan[plan_first[f] .. plan_first[f + 1]) (from lepb200_host_mux_plan).  The files are
// written back to back (16-byte aligned starts, like the device buffer) into out; off[f] / len[f] say where.
namespace {
struct GatherArgs { const GatherPiece* pieces; uint32_t n; uint8_t* out; };
void gather_body(void* p) { const GatherArgs& a = *static_cast<const GatherArgs*>(p); lep_gather_kernel(a.pieces, a.n, a.out); }
}  // namespace

extern "C" int emu_mux_files(int nfiles, const uint8_t* const* hdr, const size_t* hlen, const int* nseg, const lepb200_stream* streams,
                             const lepb200_mux_packet* plan, const uint32_t* plan_first, int grid, uint8_t* out, size_t cap, size_t* off, size_t* len) {
    if (nfiles <= 0 || !hdr || !hlen || !nseg || !streams || !plan || !plan_first || !out) return LEPB200_ERR_INVALID;
    // stream arena: 256-byte aligned starts and 256 bytes of slack like d_streams; poisoned so that a byte taken from outside a
    // stream shows
    size_t arena = 256, nstreams = 0;
    for (int f = 0; f < nfiles; ++f) for (int k = 0; k < nseg[f]; ++k) arena += align_up((size_t)streams[nstreams++].len + 16, 256);
    std::vector<uint8_t> sbuf(arena + 512, 0xEE);
    uint8_t* sbase = reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)sbuf.data(), 256));
    size_t lit_total = 0;
    for (int f = 0; f < nfiles; ++f) lit_total += align_up(hlen[f] + 4, 16);
    std::vector<uint8_t> lit(lit_total + 512, 0xDD);
    uint8_t* lbase = reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)lit.data(), 256));
    std::vector<GatherPiece> pieces;
    size_t spos = 0, lpos = 0, total = 0, si = 0;
    for (int f = 0; f < nfiles; ++f) {
        unsigned long long saddr[LEPB200_MAX_SEGMENTS];
        if (nseg[f] < 1 || nseg[f] > LEPB200_MAX_SEGMENTS) return LEPB200_ERR_INVALID;
        for (int k = 0; k < nseg[f]; ++k, ++si) {
            if (streams[si].len) memcpy(sbase + spos, streams[si].data, (size_t)streams[si].len);
            saddr[k] = (unsigned long long)(uintptr_t)(sbase + spos);
            spos += align_up((size_t)streams[si].len + 16, 256);
        }
        memcpy(lbase + lpos, hdr[f], hlen[f]);
        total = align_up(total, 16);
        off[f] = total;
        len[f] = gather_file_pieces(plan + plan_first[f], plan_first[f + 1] - plan_first[f], saddr, (unsigned long long)(uintptr_t)(lbase + lpos),
                                    lbase + lpos, hlen[f], total, pieces);
        total += len[f];
        lpos += align_up(hlen[f] + 4, 16);
    }
    if (total > cap) return LEPB200_ERR_NOMEM;
    std::vector<uint8_t> dense(total + 512, 0xCC);
    uint8_t* dbase = reinterpret_cast<uint8_t*>(align_up((size_t)(uintptr_t)dense.data(), 256));
    GatherArgs a{pieces.data(), (uint32_t)pieces.size(), dbase};
    emu::launch((unsigned)std::max(1, grid), GATHER_WARPS * 32, gather_body, &a);
    memcpy(out, dbase, total);
    return 0;
}


// ---- baseline Huffman ENCODE for the way back (lep_huffenc.cu): the jobs of lepb200_huffman_encode_resident
// (plan_huffman_encode) for one image whose planes lie in the caller's memory, one launch over all thread-segments.
// planes[c] = coefficient plane of component c (AlignedBlock layout), bch[c] / bcv[c] = its blocks per row / rows; out
// receives im->scan_bytes bytes.  reverse = 1 runs the launch's CTAs and threads in reverse order (emu::g_reverse).  Per
// segment (each output optional): status, first byte it wrote, bytes produced, Adler-32 of those bytes.
namespace {
struct HEncArgs { const HEncImage* images; HEncSeg* segs; int nseg; const HEncTable* tables; };
void henc_body(void* p) { const HEncArgs& a = *static_cast<const HEncArgs*>(p); lep_huffencode_kernel(a.images, a.segs, a.nseg, a.tables); }
}  // namespace

extern "C" int emu_huffman_encode(const lepb200_henc_image* im, int ncmp, int mcuv, const int16_t* const* planes, const int* bch, const int* bcv,
                                  int reverse, uint8_t* out, int32_t* seg_status, uint32_t* seg_off, uint32_t* seg_produced, uint32_t* seg_adler) {
    if (!im || !planes || !bch || !bcv || !out || ncmp < 1 || ncmp > 3) return LEPB200_ERR_INVALID;
    ImageDesc g;
    memset(&g, 0, sizeof(g));
    g.ncmp = ncmp; g.mcuv = mcuv;
    for (int c = 0; c < ncmp; ++c) { g.bch[c] = bch[c]; g.bcv[c] = bcv[c]; g.plane[c] = (unsigned long long)(uintptr_t)planes[c]; }
    lepb200_henc_image job = *im;
    HuffEncodePlan p;
    plan_huffman_encode(p, &job, 1, &g);
    if (p.segs.empty()) return LEPB200_ERR_INVALID;                  // nothing to encode, or a job the kernel does not take
    std::vector<uint8_t> ov;
    uint8_t* obase = host_arena(ov, p.total, 0xA5);
    p.images[0].out += (unsigned long long)(uintptr_t)obase;
    HEncArgs a{p.images.data(), p.segs.data(), (int)p.segs.size(), p.tabs.tabs.data()};
    emu::g_reverse = reverse != 0;
    emu::launch((unsigned)((p.segs.size() + HENC_WARPS - 1) / HENC_WARPS), HENC_WARPS * 32, henc_body, &a);
    emu::g_reverse = false;
    memcpy(out, obase, job.scan_bytes);
    for (size_t k = 0; k < p.segs.size(); ++k) {
        const HEncSeg& sg = p.segs[k];
        if (seg_status) seg_status[k] = sg.status;
        if (seg_off) seg_off[k] = sg.out_off;
        if (seg_produced) seg_produced[k] = sg.produced;
        if (seg_adler) seg_adler[k] = sg.adler;
    }
    return 0;
}
