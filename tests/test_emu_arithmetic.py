"""The two arithmetic shortcuts of the coder kernels, proved over their whole input domains on the CPU.

lep_common.cuh and lep_predict.cuh are compiled as host C++ through the warp emulator's shim (tests/emu/cuda_shim.h), as
test_emu_model_interleave.py does, and every input of each helper is checked:

- branch_prob: floor((c0 << 8) / (c0 + c1)) by a multiply-high with a 512-entry reciprocal table (filled as the kernels
  fill it, r[s] = ceil(2^32 / s)), for all 65 536 branch words, the special (1, 255) state of 0xff in the low byte
  included;
- branch_update: the packed-word form of Branch::record_obs_and_update, for every word and both bits, against the
  oracle's transition (oracle/lepton_oracle.c, branch.hh:82-100), probabilities included;
- div_trunc_small: truncating n / d through a float reciprocal and one correction step, for every divisor 1..65535 and
  n = k d - 1, k d, k d + 1 of both signs over the whole stated domain |n| < 2^24.

On the host, __umulhi is exact and the shim's __uint2float_rz / __frcp_rn are IEEE round-toward-zero conversion and
round-to-nearest reciprocal.  The proof carries over to the device only as far as the device's cvt.rz.f32.u32 and
rcp.rn.f32 are IEEE-exact for these inputs, which PTX specifies for both.
"""
import ctypes
import os
import subprocess

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
EMU = os.path.join(ROOT, "tests", "emu")
CSRC = os.path.join(ROOT, "lepton_b200", "csrc")

KERNEL_SRC = r"""
#include "cuda_shim.h"
#include "%s"
using namespace lepb200;
// the reciprocal table of lep_decode.cu / lep_decode_g2.cu / lep_encode.cu
static uint32_t rcp_entry(int i) { return i < 2 ? 0u : (uint32_t)((0x100000000ull + i - 1) / i); }
extern "C" void all_probs(uint32_t* out) {
    uint32_t rcp[512];
    for (int i = 0; i < 512; ++i) rcp[i] = rcp_entry(i);
    for (uint32_t w = 0; w < 65536; ++w) out[w] = branch_prob(w, rcp);
}
extern "C" void all_updates(uint32_t* out) {
    for (uint32_t w = 0; w < 65536; ++w) for (uint32_t b = 0; b < 2; ++b) out[2 * w + b] = branch_update(w, b);
}
// Mismatches of div_trunc_small(n, d) against n / d for d in [d0, d1) and n = +-(k d + e), e in {-1, 0, 1}, |n| < 2^24;
// *checked = the number of (n, d) pairs.
extern "C" uint64_t div_mismatches(int d0, int d1, uint64_t* checked) {
    const long long lim = 1ll << 24;
    uint64_t bad = 0, n_checked = 0;
    for (int d = d0; d < d1; ++d) {
        for (long long k = 0; k * d - 1 < lim; ++k) {
            for (int e = -1; e <= 1; ++e) {
                const long long m = k * d + e;
                if (m < 0 || m >= lim) continue;
                for (int sgn = -1; sgn <= 1; sgn += 2) {
                    const int n = (int)(sgn * m);
                    bad += div_trunc_small(n, d) != n / d;
                    ++n_checked;
                }
            }
        }
    }
    *checked = n_checked;
    return bad;
}
"""

ORACLE_SRC = r"""
#include "%s"
/* Branch words as the kernels pack them (low byte c0 - 1, or 0xff for the special (1, 255) state whose probability is 0;
   high byte c1 - 1) through the oracle's transition: out[2 w + obs] = new word, p[2 w + obs] = new probability, for the
   words that are states (c0, c1 in 1..255, and the special one); other words get 0xffffffff. */
void oracle_updates(uint32_t* out, uint32_t* p) {
    for (uint32_t w = 0; w < 65536; ++w) {
        const uint32_t lo = w & 0xff, hi = w >> 8;
        for (int obs = 0; obs < 2; ++obs) {
            out[2 * w + obs] = p[2 * w + obs] = 0xffffffffu;
            if (hi == 0xff || (lo == 0xff && hi != 0xfe)) continue;
            Branch b;
            if (lo == 0xff) { b.c0 = 1; b.c1 = 255; b.p = 0; }
            else { b.c0 = (uint8_t)(lo + 1); b.c1 = (uint8_t)(hi + 1); b.p = (uint8_t)(((unsigned)b.c0 << 8) / ((unsigned)b.c0 + b.c1)); }
            branch_update(&b, obs);
            const int special = b.c0 == 1 && b.c1 == 255 && b.p == 0;
            out[2 * w + obs] = special ? 0xfeffu : (uint32_t)(b.c0 - 1) | ((uint32_t)(b.c1 - 1) << 8);
            p[2 * w + obs] = b.p;
        }
    }
}
"""


@pytest.fixture(scope="module")
def libs(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("arith")
    k_src, o_src = tmp / "kernels.cc", tmp / "oracle.c"
    k_src.write_text(KERNEL_SRC % os.path.join(CSRC, "lep_predict.cuh"))
    o_src.write_text(ORACLE_SRC % os.path.join(ROOT, "oracle", "lepton_oracle.c"))
    k_so, o_so = str(tmp / "kernels.so"), str(tmp / "oracle.so")
    subprocess.check_call(["g++", "-O2", "-std=c++17", "-shared", "-fPIC", "-x", "c++", "-I", EMU, "-I", os.path.join(EMU, "fake"),
                           "-Wno-unknown-pragmas", "-o", k_so, str(k_src)])
    subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-fwrapv", "-w", "-o", o_so, str(o_src)])
    k, o = ctypes.CDLL(k_so), ctypes.CDLL(o_so)
    k.div_mismatches.restype = ctypes.c_uint64
    k.div_mismatches.argtypes = [ctypes.c_int, ctypes.c_int, ctypes.POINTER(ctypes.c_uint64)]
    return k, o


def test_branch_prob_reciprocal_division_for_every_word(libs):
    k, _ = libs
    got = np.zeros(65536, np.uint32)
    k.all_probs(got.ctypes.data_as(ctypes.c_void_p))
    w = np.arange(65536, dtype=np.uint64)
    lo, hi = w & 0xff, w >> 8
    want = np.where(lo == 0xff, 0, ((lo + 1) << 8) // (lo + hi + 2)).astype(np.uint32)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(hex(int(x)), int(got[x]), int(want[x])) for x in bad[:8]]
    assert got[0xfeff] == 0 and got[0x00fe] == 255 and got[0xfe00] == 1     # special state, (255, 1), plain (1, 255)


def test_branch_update_matches_the_oracle_transition(libs):
    k, o = libs
    got = np.zeros(2 * 65536, np.uint32)
    want = np.zeros(2 * 65536, np.uint32)
    want_p = np.zeros(2 * 65536, np.uint32)
    k.all_updates(got.ctypes.data_as(ctypes.c_void_p))
    o.oracle_updates(want.ctypes.data_as(ctypes.c_void_p), want_p.ctypes.data_as(ctypes.c_void_p))
    states = want != 0xffffffff
    assert np.count_nonzero(states) == 2 * (255 * 255 + 1)
    bad = np.flatnonzero(states & (got != want))
    assert bad.size == 0, [(hex(int(x) // 2), int(x) % 2, hex(int(got[x])), hex(int(want[x]))) for x in bad[:8]]
    # the probability the kernels read from the new word is the oracle's
    probs = np.zeros(65536, np.uint32)
    k.all_probs(probs.ctypes.data_as(ctypes.c_void_p))
    assert np.array_equal(probs[got[states]], want_p[states])
    assert got[2 * 0xfe00 + 1] == 0xfeff          # c1 overflows while c0 == 1: the special state
    assert got[2 * 0x00fe + 0] == 0x00fe          # c0 overflows while c1 == 1: stays (255, 1)


def test_div_trunc_small_for_every_divisor_around_every_multiple(libs):
    k, _ = libs
    checked = ctypes.c_uint64(0)
    bad = k.div_mismatches(1, 65536, ctypes.byref(checked))
    assert bad == 0
    assert checked.value > 6 * (1 << 24) * 10         # sum over d of 6 * 2^24 / d
