// emu_ans_kernels.cc -- the decode kernels with the rANS coder of container version 3 on the CPU under the warp emulator of
// cuda_shim.h (test infrastructure), next to emu_kernels.cc: the same kernel sources, the planner of the library
// (lep_plan.cuh, with a coder per image) and the launch split of lepb200_decode_launch (the bool-coded segments of a batch in
// one launch, the rANS-coded ones in another).
#include <algorithm>
#include <cstdlib>
#include <vector>

#include "cuda_shim.h"
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
    bool ans;                        // the launch's segments are rANS-coded (CODER_ANS)
    const ImageDesc* images; SegDesc* segs; int nseg; const int* order; int* counter;
    uint16_t* models; uint8_t* rows; size_t row_stride;
};

template <class WarpReader, class GroupCoder> void kernel_body_coder(const LaunchArgs& a) {
    if (a.kernel == 0) lep_decode_kernel<WarpReader>(a.images, a.segs, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 201) lep_decode_g2_kernel<1, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 202) lep_decode_g2_kernel<2, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 204) lep_decode_g2_kernel<4, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 208) lep_decode_g2_kernel<8, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else if (a.kernel == 216) lep_decode_g2_kernel<16, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
    else lep_decode_g2_kernel<32, GroupCoder>(a.images, a.segs, 0, a.nseg, a.order, a.counter, a.models, a.rows, a.row_stride);
}

void kernel_body(void* p) {
    const LaunchArgs& a = *static_cast<const LaunchArgs*>(p);
    if (a.ans) kernel_body_coder<AnsReader, G2Ans>(a);
    else kernel_body_coder<BoolReader, G2Bool>(a);
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
// reverse = 1 runs the launch's CTAs and threads in reverse order (emu::g_reverse).  coders (optional): the entropy coder of
// each image's streams (LEPB200_CODER_*); as in lepb200_decode_launch, the bool-coded segments of the batch are decoded by one
// launch and the rANS-coded ones by another, both of the given kernel.
extern "C" int emu_decode_images_coded(int kernel, int grid_cap, int reverse, const lepb200_image* images, int nimages, const lepb200_stream* in,
                                       const uint8_t* coders, int32_t* status_out, uint64_t* ndecisions_out) {
    const int gl = kernel % 100;
    const bool group = kernel / 100 == 2 && (gl == 1 || gl == 2 || gl == 4 || gl == 8 || gl == 16 || gl == 32);
    if (!in || (kernel != 0 && !group)) return LEPB200_ERR_INVALID;
    BatchPlan b;
    if (plan_batch(b, images, nimages, false, in, coders)) return LEPB200_ERR_INVALID;
    const int nseg = (int)b.segs.size();
    // planes start zeroed like the device arena; the stream arena is not cleared: whatever is behind a stream must not matter
    std::vector<uint8_t> pv, sv;
    uint8_t* pbase = host_arena(pv, b.plane_total, 0);
    uint8_t* sbase = host_arena(sv, b.stream_total, 0xA5);
    for (int s = 0; s < nseg; ++s) if (in[s].len) memcpy(sbase + b.segs[s].stream, in[s].data, (size_t)in[s].len);
    rebase(b, pbase, sbase);
    std::vector<SegDesc>& segs = b.segs;
    for (int part = 0; part < 2; ++part) {
        const int first = part == 0 ? 0 : b.order_ans, n = part == 0 ? b.order_ans : nseg - b.order_ans;
        if (n == 0) continue;
        LaunchArgs a;
        a.kernel = kernel; a.ans = part == 1; a.images = b.images.data(); a.segs = segs.data(); a.nseg = n; a.order = b.order.data() + first;
        a.row_stride = b.row_stride;
        int counter = 0;
        a.counter = &counter;
        unsigned grid, block;
        size_t group_slots = 0;
        if (group) {
            // 200 + G: lep_decode_g2_kernel<G>; grid_cap > 0 limits the CTAs so that groups take several segments from the queue
            int warps, per_warp;
            group_shape(kernel % 100, warps, per_warp);
            grid = (unsigned)((n + warps * per_warp - 1) / (warps * per_warp));
            if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
            block = (unsigned)warps * 32;
            group_slots = (size_t)grid * warps * per_warp;
        } else {
            grid = (unsigned)((n + DEC_WARPS_PER_CTA - 1) / DEC_WARPS_PER_CTA);
            if (grid_cap > 0) grid = std::min(grid, (unsigned)grid_cap);
            block = DEC_WARPS_PER_CTA * 32;
        }
        const size_t slots = kernel == 0 ? (size_t)grid * DEC_WARPS_PER_CTA : (size_t)n;
        std::vector<uint16_t> models(slots * M_TOTAL, kernel == 0 ? 0x5a5a : 0);       // thread / group kernels: zero fill before the launch; the warp kernel clears its own
        std::vector<uint8_t> rows((group ? group_slots : slots) * b.row_stride, 0);
        a.models = models.data(); a.rows = rows.data();
        emu::g_reverse = reverse != 0;
        emu::launch(grid, block, kernel_body, &a);
        emu::g_reverse = false;
    }
    for (int i = 0; i < nimages; ++i)
        for (int c = 0; c < images[i].ncmp; ++c)
            memcpy(images[i].planes[c], reinterpret_cast<const void*>(b.images[i].plane[c]), b.plane_bytes[(size_t)i * 3 + c]);
    for (int s = 0; s < nseg; ++s) {
        if (status_out) status_out[s] = segs[s].status;
        if (ndecisions_out) ndecisions_out[s] = (uint64_t)segs[s].ndecisions_lo | ((uint64_t)segs[s].ndecisions_hi << 32);
    }
    return 0;
}

