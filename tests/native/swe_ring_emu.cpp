// Host emulation of the pair schedule's ring launch as one launch (csrc/b2_swe_ca.cu: swe_ca_bulk_step
// over the table of the four ring windows, blockIdx.y the window), on top of swe_pair_emu.cpp, whose
// entry points this library also exports.
// Build: g++ -O1 -ffp-contract=off -shared -fPIC -I csrc -I $CUDA/include tests/native/swe_ring_emu.cpp
#include "swe_pair_emu.cpp"

extern "C" {

// the ring launch: the windows of swe_pair_emu.cpp's window() 2 .. 5 as one table, blocks of
// CA_BULK_WARPS warps, blocks past a window's warps idle
void emu_ca_ring(const B2SweParams* p, const EmuIO* e, int reverse) {
  CABulkArgs a = window(p, 2, 2);
  set_io(a, e);
  CAWin win[4];
  long long blocks = 0;
  for (int y = 0; y < 4; ++y) {
    win[y] = window(p, 2 + y, 2);
    const long long nb = (ca_bulk_warps(win[y]) + CA_BULK_WARPS - 1) / CA_BULK_WARPS;
    blocks = nb > blocks ? nb : blocks;
  }
  static CABulkLane L[32];
  bool yes[32];
  for (int l = 0; l < 32; ++l) yes[l] = true;
  const long long nw = 4 * blocks * CA_BULK_WARPS;
  for (long long k = 0; k < nw; ++k) {
    const long long t = reverse ? nw - 1 - k : k;
    const CAWin& g = win[t / (blocks * CA_BULK_WARPS)];
    const int wi = (int)(t % (blocks * CA_BULK_WARPS));
    if (wi >= ca_bulk_warps(g)) continue;
    int s, en;
    ca_bulk_rows(g, wi / g.wcols, s, en);
    for (int l = 0; l < 32; ++l) {
      L[l].store = ca_bulk_lane(g, wi % g.wcols, l, L[l].i0);
      ca_bulk_begin(a, L[l], s);
    }
    for (int r = s - 2; r <= en; ++r) warp_row<false, false>(a, L, r, s, en, nullptr, yes, yes);
  }
}

}  // extern "C"
