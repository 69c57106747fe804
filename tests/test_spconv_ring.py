"""The stage / parity arithmetic of the pipelined sparse convolution (csrc/spconv_ring.h), walked on the host.

A small C++ driver plays producer and consumer of spconv_tc_kernel against two-phase barriers that, like mbarriers,
only compare parities: over runs of tiles with mixed chunk counts, under random interleavings, both sides must agree
on which chunk a stage holds, every wait must pass on exactly the completion it meant, the producer is never more
than kStages chunks ahead, and a tile's parked out rows are not overwritten before its epilogue has read them.
"""
import os
import shutil
import subprocess

import pytest

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), 'deepglobalregistration_b200', 'csrc')

DRIVER = r'''
#include <cstdio>
#include <cstdlib>
#include <vector>
#include "spconv_ring.h"
using namespace spconv_ring;
#define CHECK(c) do { if (!(c)) { std::printf("FAILED %s (line %d)\n", #c, __LINE__); return 1; } } while (0)

int main(int argc, char** argv) {
  if (argc > 1 && argv[1][0] == 'r') {                  // tile_run n_tiles resident
    std::printf("%d\n", tile_run(std::atoi(argv[2]), std::atoi(argv[3])));
    return 0;
  }
  unsigned seed = (unsigned)std::atoi(argv[1]);
  std::vector<int> chunks;                              // chunk count of every tile of the run
  for (int i = 2; i < argc; ++i) chunks.push_back(std::atoi(argv[i]));
  const int n = (int)chunks.size();
  unsigned full[kStages] = {}, empty[kStages] = {};     // completed phases of each barrier
  long held[kStages];                                   // chunk a stage holds
  int slot[kIdxSlots];                                  // tile whose out rows a slot holds
  for (int s = 0; s < kStages; ++s) held[s] = -1;
  for (int s = 0; s < kIdxSlots; ++s) slot[s] = -1;
  auto passes = [](unsigned phases, unsigned parity) { return (phases & 1u) != parity; };
  // producer position (tile, chunk, running chunk), consumer position, chunks released, tiles drained
  int pt = 0, pc = 0, ct = 0, cc = 0, drained = 0;
  unsigned pg = 0, cg = 0, released = 0;
  while (ct < n) {
    seed = seed * 1664525u + 1013904223u;
    bool moved = false;
    for (int attempt = 0; attempt < 2 && !moved; ++attempt) {
      const bool producer = (((seed >> 16) & 1u) != 0) != (attempt == 1);
      if (producer && pt < n) {
        const int s = stage_of(pg);
        if (pg >= (unsigned)kStages) {
          if (!passes(empty[s], empty_parity(pg))) continue;
          CHECK(empty[s] == pg / kStages);              // the completion it waited for, not a later one
        }
        if (pc == 0) {
          const int old = slot[idx_slot(pt)];
          CHECK(old < 0 || old < drained);              // that tile's epilogue has read its rows
          slot[idx_slot(pt)] = pt;
        }
        held[s] = pg;
        ++full[s];
        ++pg;
        CHECK(pg - released <= (unsigned)kStages);
        if (++pc == chunks[pt]) { pc = 0; ++pt; }
        moved = true;
      } else if (!producer) {
        const int s = stage_of(cg);
        if (!passes(full[s], full_parity(cg))) continue;
        CHECK(full[s] == cg / kStages + 1);
        CHECK(held[s] == (long)cg);
        if (cc > 0) { ++empty[stage_of(cg - 1)]; ++released; }      // wgmma_wait<1>: the previous chunk retired
        ++cg;
        if (++cc == chunks[ct]) {                                   // wgmma_wait<0>, then the epilogue
          ++empty[stage_of(cg - 1)]; ++released;
          CHECK(slot[idx_slot(ct)] == ct);
          cc = 0; ++ct; ++drained;
        }
        moved = true;
      }
    }
    CHECK(moved);                                       // neither side can move: the ring would hang
  }
  CHECK(pt == n && pg == cg && released == cg);
  std::printf("ok %u\n", cg);
  return 0;
}
'''


@pytest.fixture(scope='module')
def driver(tmp_path_factory):
  cxx = shutil.which('g++') or shutil.which('c++')
  if cxx is None:
    pytest.skip('no host C++ compiler')
  d = tmp_path_factory.mktemp('ring')
  (d / 'ring.cc').write_text(DRIVER)
  exe = str(d / 'ring')
  subprocess.run([cxx, '-std=c++17', '-O1', '-I', CSRC, str(d / 'ring.cc'), '-o', exe], check=True)
  return exe


@pytest.mark.parametrize('chunks', [
    [1], [4], [1] * 9, [2] * 8, [3] * 8, [4] * 8,          # one tile; odd counts carry the ring position over
    [1, 2, 3, 4, 4, 3, 2, 1], [3, 1, 1, 3, 2, 1, 4, 1, 1, 1, 3, 3], [8, 1, 8, 1, 3],
])
def test_ring_walk(driver, chunks):
  for seed in range(20):
    r = subprocess.run([driver, str(seed)] + [str(c) for c in chunks], capture_output=True, text=True)
    assert r.returncode == 0 and r.stdout.split() == ['ok', str(sum(chunks))], (seed, r.stdout, r.stderr)


def test_tile_run(driver):
  run = lambda n, resident: int(subprocess.run([driver, 'r', str(n), str(resident)], capture_output=True,
                                               text=True, check=True).stdout)
  assert run(1, 132) == 1 and run(263, 132) == 1 and run(527, 132) == 1      # the grid covers the device twice first
  assert run(528, 132) == 2 and run(3 * 264, 132) == 3
  assert run(21000, 132) == run(10 ** 6, 264) == 8                            # the cap
