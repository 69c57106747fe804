// Ring arithmetic of the pipelined tensor-core sparse convolution (spconv_tc.cu), free of CUDA types so that a
// host program can walk it (tests/test_spconv_ring.py).
//
// A CTA works through a run of tiles; every tile is n_chunks K-chunks, and chunk number g of the run (a counter
// that keeps running across tile boundaries) lives in stage g % stages.  A stage has two mbarriers: `full`
// (producer -> consumers: operands have landed) and `empty` (consumers -> producer: the MMAs that read the stage
// have retired).  Both complete one phase per use of the stage, so the parity a waiter passes to
// mbarrier.try_wait is the use count's lowest bit.
#pragma once

#if defined(__CUDACC__)
#define DGR_RING_HD __host__ __device__ __forceinline__
#else
#define DGR_RING_HD inline
#endif

namespace spconv_ring {

constexpr int kStages = 2;
// out rows of a tile are parked per tile, not per stage: while the consumers drain tile t the producer may already
// have filled the first chunk of up to kStages later tiles
constexpr int kIdxSlots = kStages + 1;
// most tiles one CTA works through: long enough to hide a tile's head and tail behind its neighbours, short
// enough that the SMs keep turning over for the other streams' latency-bound kernels
constexpr int kMaxRun = 8;

DGR_RING_HD int stage_of(unsigned g) { return (int)(g % kStages); }
// consumers, before the MMAs of chunk g: wait for the (g / kStages)-th completion of full[stage_of(g)]
DGR_RING_HD unsigned full_parity(unsigned g) { return (g / kStages) & 1u; }
// producer, before it overwrites the stage with chunk g >= kStages: wait until chunk g - kStages has been retired,
// the (g / kStages - 1)-th completion of empty[stage_of(g)]
DGR_RING_HD unsigned empty_parity(unsigned g) { return (g / kStages - 1u) & 1u; }
DGR_RING_HD int idx_slot(unsigned tile) { return (int)(tile % kIdxSlots); }

// tiles per CTA for a launch of n_tiles on a device that holds `resident` CTAs of the kernel at once: one while
// the grid would not cover the device kMinWaves times, then growing with the launch up to kMaxRun.  Measured on
// the benchmark with four pairs in flight (DESIGN 3): 2 waves give more pairs/s than 8, although single mid-size
// launches, timed alone, lose to the wave tail at 2
constexpr int kMinWaves = 2;
DGR_RING_HD int tile_run(int n_tiles, int resident) {
  const int r = n_tiles / (kMinWaves * (resident > 0 ? resident : 1));
  return r < 1 ? 1 : (r > kMaxRun ? kMaxRun : r);
}

}  // namespace spconv_ring
