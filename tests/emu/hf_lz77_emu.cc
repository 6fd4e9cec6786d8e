// TEST INFRASTRUCTURE — NOT PART OF THE PRODUCT.
//
// The host emulation of the thread-per-stream HF coefficient kernel (emu_backend.cc) built with a count of the values
// its LZ77 streams take from copies, so that tests/test_hf_lz77.py can show that copies really ran: make -f hf_lz77.mk.
#include <atomic>
#include <cstdint>

namespace {
std::atomic<uint64_t> g_hf_lz77_copied{0};
}  // namespace
#define JXLB_LANE_LZ77_COPIED(n) (::g_hf_lz77_copied += (n))
#include "emu_backend.cc"

// values the emulated HF streams took from LZ77 copies so far
extern "C" uint64_t jxle_hf_lz77_copied() { return g_hf_lz77_copied.load(); }
// hf_lz77_window_entries (launch_tables.cc): the LZ77 window of one HF stream, for groups of `group_dim` pixels
extern "C" uint64_t jxle_hf_lz77_window_entries(uint32_t group_dim) { return jxlb::hf_lz77_window_entries(group_dim); }
