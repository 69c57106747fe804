// RGB-D fusion into a sparse TSDF volume and its marching-cubes mesh: open3d's legacy ScalableTSDFVolume
// (integrate, extract_triangle_mesh) as util/integration.py drives it.  oracle/tsdf.py is the arithmetic contract;
// every floating-point operation here is an explicit round-to-nearest intrinsic in the order the oracle states, so
// nothing contracts to an FMA and the state and the mesh are the oracle's bit for bit.
//
// Volume: units of 16^3 voxels, keyed by unit coordinate in a persistent open-addressing table (fixed 3 x 21-bit
// packing: the volume grows, so there is no min/max key spec) that maps a key to the unit's slot; slots number units in
// order of first touch.  Slabs are structure-of-arrays per slot: tsdf[4096], weight[4096], colour[3][4096] (fp32).
//
//   dgr_tsdf_touch       a thread per sampled pixel writes its candidate units (side^3 per sample, a sentinel where
//                        none), dgr_unique_first keeps first occurrences, survivors are looked up; new ones are
//                        flagged and ranked by dgr_scan_counts + dgr_select_first, take slots n_total + rank and are
//                        inserted.  touched[] lists the slots in first-occurrence order; counts = (n_touched, n_total).
//   dgr_tsdf_integrate   one CTA per touched unit, a thread per voxel at t + 256 k: coalesced slab reads and writes;
//                        each voxel has one writer per frame, so no atomics.
//   dgr_tsdf_extract_*   count: classify every cube of a unit over its +1 halo (7 neighbour units through the table,
//                        in shared memory), OR each sign-changing edge of a kept cube into its owner voxel's bit (the
//                        edge's lower endpoint, which may lie in a +1 neighbour; bits commute, so the masks are the
//                        same on every run), per-unit triangle counts; popcount word prefixes and vertex counts per
//                        unit; two count scans.  write: vertices by (slot, voxel, axis) from the masks, triangles by
//                        (slot, voxel, table order) with a block scan per 256 voxels.
//   dgr_tsdf_raycast     a thread per pixel marches its ray through the unit table (a missing unit is jumped past its
//                        exit plane, a known voxel by its tsdf distance, an unknown one by a voxel) to the first
//                        + to - crossing; depth, and for RGB8 the trilinear colour and its intensity.  Read-only.
#include <limits.h>
#include <math.h>
#include <math_constants.h>
#include <stdio.h>

#include "common.cuh"

namespace {

constexpr int kRes = DGR_TSDF_RES;
constexpr int kVox = kRes * kRes * kRes;     // 4096 voxels per unit
constexpr int kThreads = 256;
constexpr int kPerThread = kVox / kThreads;  // 16
constexpr int kHalo = kRes + 1;              // 17: a unit plus its +1 layer
constexpr int kHaloN = kHalo * kHalo * kHalo;
constexpr int kMaskWords = kVox / 32;        // 128 words per axis per unit
constexpr int kCoordBias = 1 << 20;          // unit coordinate + bias in [0, 2^21)
constexpr int kSentinel = DGR_TSDF_COORD_MAX + 1;

// Lorensen / Bourke marching-cubes triangle table, corners 0..7 = (000, 100, 110, 010, 001, 101, 111, 011); oracle/tsdf.py
// restates it.  One text, instantiated for the device and for dgr_tsdf_mc_tables.
#define DGR_MC_TRI_TABLE {                                                                                         \
  {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,8,3,9,8,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,1,2,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,2,10,0,2,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,8,3,2,10,8,10,9,8,-1,-1,-1,-1,-1,-1,-1}, \
  {3,11,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,11,2,8,11,0,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,9,0,2,3,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,11,2,1,9,11,9,8,11,-1,-1,-1,-1,-1,-1,-1}, \
  {3,10,1,11,10,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,10,1,0,8,10,8,11,10,-1,-1,-1,-1,-1,-1,-1}, {3,9,0,3,11,9,11,10,9,-1,-1,-1,-1,-1,-1,-1}, {9,8,10,10,8,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,3,0,7,3,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,8,4,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,1,9,4,7,1,7,3,1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,10,8,4,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,4,7,3,0,4,1,2,10,-1,-1,-1,-1,-1,-1,-1}, {9,2,10,9,0,2,8,4,7,-1,-1,-1,-1,-1,-1,-1}, {2,10,9,2,9,7,2,7,3,7,9,4,-1,-1,-1,-1}, \
  {8,4,7,3,11,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,4,7,11,2,4,2,0,4,-1,-1,-1,-1,-1,-1,-1}, {9,0,1,8,4,7,2,3,11,-1,-1,-1,-1,-1,-1,-1}, {4,7,11,9,4,11,9,11,2,9,2,1,-1,-1,-1,-1}, \
  {3,10,1,3,11,10,7,8,4,-1,-1,-1,-1,-1,-1,-1}, {1,11,10,1,4,11,1,0,4,7,11,4,-1,-1,-1,-1}, {4,7,8,9,0,11,9,11,10,11,0,3,-1,-1,-1,-1}, {4,7,11,4,11,9,9,11,10,-1,-1,-1,-1,-1,-1,-1}, \
  {9,5,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,5,4,0,8,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,5,4,1,5,0,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,5,4,8,3,5,3,1,5,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,10,9,5,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,1,2,10,4,9,5,-1,-1,-1,-1,-1,-1,-1}, {5,2,10,5,4,2,4,0,2,-1,-1,-1,-1,-1,-1,-1}, {2,10,5,3,2,5,3,5,4,3,4,8,-1,-1,-1,-1}, \
  {9,5,4,2,3,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,11,2,0,8,11,4,9,5,-1,-1,-1,-1,-1,-1,-1}, {0,5,4,0,1,5,2,3,11,-1,-1,-1,-1,-1,-1,-1}, {2,1,5,2,5,8,2,8,11,4,8,5,-1,-1,-1,-1}, \
  {10,3,11,10,1,3,9,5,4,-1,-1,-1,-1,-1,-1,-1}, {4,9,5,0,8,1,8,10,1,8,11,10,-1,-1,-1,-1}, {5,4,0,5,0,11,5,11,10,11,0,3,-1,-1,-1,-1}, {5,4,8,5,8,10,10,8,11,-1,-1,-1,-1,-1,-1,-1}, \
  {9,7,8,5,7,9,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,3,0,9,5,3,5,7,3,-1,-1,-1,-1,-1,-1,-1}, {0,7,8,0,1,7,1,5,7,-1,-1,-1,-1,-1,-1,-1}, {1,5,3,3,5,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {9,7,8,9,5,7,10,1,2,-1,-1,-1,-1,-1,-1,-1}, {10,1,2,9,5,0,5,3,0,5,7,3,-1,-1,-1,-1}, {8,0,2,8,2,5,8,5,7,10,5,2,-1,-1,-1,-1}, {2,10,5,2,5,3,3,5,7,-1,-1,-1,-1,-1,-1,-1}, \
  {7,9,5,7,8,9,3,11,2,-1,-1,-1,-1,-1,-1,-1}, {9,5,7,9,7,2,9,2,0,2,7,11,-1,-1,-1,-1}, {2,3,11,0,1,8,1,7,8,1,5,7,-1,-1,-1,-1}, {11,2,1,11,1,7,7,1,5,-1,-1,-1,-1,-1,-1,-1}, \
  {9,5,8,8,5,7,10,1,3,10,3,11,-1,-1,-1,-1}, {5,7,0,5,0,9,7,11,0,1,0,10,11,10,0,-1}, {11,10,0,11,0,3,10,5,0,8,0,7,5,7,0,-1}, {11,10,5,7,11,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {10,6,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {9,0,1,5,10,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,8,3,1,9,8,5,10,6,-1,-1,-1,-1,-1,-1,-1}, \
  {1,6,5,2,6,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,6,5,1,2,6,3,0,8,-1,-1,-1,-1,-1,-1,-1}, {9,6,5,9,0,6,0,2,6,-1,-1,-1,-1,-1,-1,-1}, {5,9,8,5,8,2,5,2,6,3,2,8,-1,-1,-1,-1}, \
  {2,3,11,10,6,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,0,8,11,2,0,10,6,5,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,2,3,11,5,10,6,-1,-1,-1,-1,-1,-1,-1}, {5,10,6,1,9,2,9,11,2,9,8,11,-1,-1,-1,-1}, \
  {6,3,11,6,5,3,5,1,3,-1,-1,-1,-1,-1,-1,-1}, {0,8,11,0,11,5,0,5,1,5,11,6,-1,-1,-1,-1}, {3,11,6,0,3,6,0,6,5,0,5,9,-1,-1,-1,-1}, {6,5,9,6,9,11,11,9,8,-1,-1,-1,-1,-1,-1,-1}, \
  {5,10,6,4,7,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,3,0,4,7,3,6,5,10,-1,-1,-1,-1,-1,-1,-1}, {1,9,0,5,10,6,8,4,7,-1,-1,-1,-1,-1,-1,-1}, {10,6,5,1,9,7,1,7,3,7,9,4,-1,-1,-1,-1}, \
  {6,1,2,6,5,1,4,7,8,-1,-1,-1,-1,-1,-1,-1}, {1,2,5,5,2,6,3,0,4,3,4,7,-1,-1,-1,-1}, {8,4,7,9,0,5,0,6,5,0,2,6,-1,-1,-1,-1}, {7,3,9,7,9,4,3,2,9,5,9,6,2,6,9,-1}, \
  {3,11,2,7,8,4,10,6,5,-1,-1,-1,-1,-1,-1,-1}, {5,10,6,4,7,2,4,2,0,2,7,11,-1,-1,-1,-1}, {0,1,9,4,7,8,2,3,11,5,10,6,-1,-1,-1,-1}, {9,2,1,9,11,2,9,4,11,7,11,4,5,10,6,-1}, \
  {8,4,7,3,11,5,3,5,1,5,11,6,-1,-1,-1,-1}, {5,1,11,5,11,6,1,0,11,7,11,4,0,4,11,-1}, {0,5,9,0,6,5,0,3,6,11,6,3,8,4,7,-1}, {6,5,9,6,9,11,4,7,9,7,11,9,-1,-1,-1,-1}, \
  {10,4,9,6,4,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,10,6,4,9,10,0,8,3,-1,-1,-1,-1,-1,-1,-1}, {10,0,1,10,6,0,6,4,0,-1,-1,-1,-1,-1,-1,-1}, {8,3,1,8,1,6,8,6,4,6,1,10,-1,-1,-1,-1}, \
  {1,4,9,1,2,4,2,6,4,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,1,2,9,2,4,9,2,6,4,-1,-1,-1,-1}, {0,2,4,4,2,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,3,2,8,2,4,4,2,6,-1,-1,-1,-1,-1,-1,-1}, \
  {10,4,9,10,6,4,11,2,3,-1,-1,-1,-1,-1,-1,-1}, {0,8,2,2,8,11,4,9,10,4,10,6,-1,-1,-1,-1}, {3,11,2,0,1,6,0,6,4,6,1,10,-1,-1,-1,-1}, {6,4,1,6,1,10,4,8,1,2,1,11,8,11,1,-1}, \
  {9,6,4,9,3,6,9,1,3,11,6,3,-1,-1,-1,-1}, {8,11,1,8,1,0,11,6,1,9,1,4,6,4,1,-1}, {3,11,6,3,6,0,0,6,4,-1,-1,-1,-1,-1,-1,-1}, {6,4,8,11,6,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {7,10,6,7,8,10,8,9,10,-1,-1,-1,-1,-1,-1,-1}, {0,7,3,0,10,7,0,9,10,6,7,10,-1,-1,-1,-1}, {10,6,7,1,10,7,1,7,8,1,8,0,-1,-1,-1,-1}, {10,6,7,10,7,1,1,7,3,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,6,1,6,8,1,8,9,8,6,7,-1,-1,-1,-1}, {2,6,9,2,9,1,6,7,9,0,9,3,7,3,9,-1}, {7,8,0,7,0,6,6,0,2,-1,-1,-1,-1,-1,-1,-1}, {7,3,2,6,7,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {2,3,11,10,6,8,10,8,9,8,6,7,-1,-1,-1,-1}, {2,0,7,2,7,11,0,9,7,6,7,10,9,10,7,-1}, {1,8,0,1,7,8,1,10,7,6,7,10,2,3,11,-1}, {11,2,1,11,1,7,10,6,1,6,7,1,-1,-1,-1,-1}, \
  {8,9,6,8,6,7,9,1,6,11,6,3,1,3,6,-1}, {0,9,1,11,6,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {7,8,0,7,0,6,3,11,0,11,6,0,-1,-1,-1,-1}, {7,11,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {7,6,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,8,11,7,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,1,9,11,7,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,1,9,8,3,1,11,7,6,-1,-1,-1,-1,-1,-1,-1}, \
  {10,1,2,6,11,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,2,10,3,0,8,6,11,7,-1,-1,-1,-1,-1,-1,-1}, {2,9,0,2,10,9,6,11,7,-1,-1,-1,-1,-1,-1,-1}, {6,11,7,2,10,3,10,8,3,10,9,8,-1,-1,-1,-1}, \
  {7,2,3,6,2,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {7,0,8,7,6,0,6,2,0,-1,-1,-1,-1,-1,-1,-1}, {2,7,6,2,3,7,0,1,9,-1,-1,-1,-1,-1,-1,-1}, {1,6,2,1,8,6,1,9,8,8,7,6,-1,-1,-1,-1}, \
  {10,7,6,10,1,7,1,3,7,-1,-1,-1,-1,-1,-1,-1}, {10,7,6,1,7,10,1,8,7,1,0,8,-1,-1,-1,-1}, {0,3,7,0,7,10,0,10,9,6,10,7,-1,-1,-1,-1}, {7,6,10,7,10,8,8,10,9,-1,-1,-1,-1,-1,-1,-1}, \
  {6,8,4,11,8,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,6,11,3,0,6,0,4,6,-1,-1,-1,-1,-1,-1,-1}, {8,6,11,8,4,6,9,0,1,-1,-1,-1,-1,-1,-1,-1}, {9,4,6,9,6,3,9,3,1,11,3,6,-1,-1,-1,-1}, \
  {6,8,4,6,11,8,2,10,1,-1,-1,-1,-1,-1,-1,-1}, {1,2,10,3,0,11,0,6,11,0,4,6,-1,-1,-1,-1}, {4,11,8,4,6,11,0,2,9,2,10,9,-1,-1,-1,-1}, {10,9,3,10,3,2,9,4,3,11,3,6,4,6,3,-1}, \
  {8,2,3,8,4,2,4,6,2,-1,-1,-1,-1,-1,-1,-1}, {0,4,2,4,6,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {1,9,0,2,3,4,2,4,6,4,3,8,-1,-1,-1,-1}, {1,9,4,1,4,2,2,4,6,-1,-1,-1,-1,-1,-1,-1}, \
  {8,1,3,8,6,1,8,4,6,6,10,1,-1,-1,-1,-1}, {10,1,0,10,0,6,6,0,4,-1,-1,-1,-1,-1,-1,-1}, {4,6,3,4,3,8,6,10,3,0,3,9,10,9,3,-1}, {10,9,4,6,10,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {4,9,5,7,6,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,4,9,5,11,7,6,-1,-1,-1,-1,-1,-1,-1}, {5,0,1,5,4,0,7,6,11,-1,-1,-1,-1,-1,-1,-1}, {11,7,6,8,3,4,3,5,4,3,1,5,-1,-1,-1,-1}, \
  {9,5,4,10,1,2,7,6,11,-1,-1,-1,-1,-1,-1,-1}, {6,11,7,1,2,10,0,8,3,4,9,5,-1,-1,-1,-1}, {7,6,11,5,4,10,4,2,10,4,0,2,-1,-1,-1,-1}, {3,4,8,3,5,4,3,2,5,10,5,2,11,7,6,-1}, \
  {7,2,3,7,6,2,5,4,9,-1,-1,-1,-1,-1,-1,-1}, {9,5,4,0,8,6,0,6,2,6,8,7,-1,-1,-1,-1}, {3,6,2,3,7,6,1,5,0,5,4,0,-1,-1,-1,-1}, {6,2,8,6,8,7,2,1,8,4,8,5,1,5,8,-1}, \
  {9,5,4,10,1,6,1,7,6,1,3,7,-1,-1,-1,-1}, {1,6,10,1,7,6,1,0,7,8,7,0,9,5,4,-1}, {4,0,10,4,10,5,0,3,10,6,10,7,3,7,10,-1}, {7,6,10,7,10,8,5,4,10,4,8,10,-1,-1,-1,-1}, \
  {6,9,5,6,11,9,11,8,9,-1,-1,-1,-1,-1,-1,-1}, {3,6,11,0,6,3,0,5,6,0,9,5,-1,-1,-1,-1}, {0,11,8,0,5,11,0,1,5,5,6,11,-1,-1,-1,-1}, {6,11,3,6,3,5,5,3,1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,10,9,5,11,9,11,8,11,5,6,-1,-1,-1,-1}, {0,11,3,0,6,11,0,9,6,5,6,9,1,2,10,-1}, {11,8,5,11,5,6,8,0,5,10,5,2,0,2,5,-1}, {6,11,3,6,3,5,2,10,3,10,5,3,-1,-1,-1,-1}, \
  {5,8,9,5,2,8,5,6,2,3,8,2,-1,-1,-1,-1}, {9,5,6,9,6,0,0,6,2,-1,-1,-1,-1,-1,-1,-1}, {1,5,8,1,8,0,5,6,8,3,8,2,6,2,8,-1}, {1,5,6,2,1,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,3,6,1,6,10,3,8,6,5,6,9,8,9,6,-1}, {10,1,0,10,0,6,9,5,0,5,6,0,-1,-1,-1,-1}, {0,3,8,5,6,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {10,5,6,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {11,5,10,7,5,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {11,5,10,11,7,5,8,3,0,-1,-1,-1,-1,-1,-1,-1}, {5,11,7,5,10,11,1,9,0,-1,-1,-1,-1,-1,-1,-1}, {10,7,5,10,11,7,9,8,1,8,3,1,-1,-1,-1,-1}, \
  {11,1,2,11,7,1,7,5,1,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,1,2,7,1,7,5,7,2,11,-1,-1,-1,-1}, {9,7,5,9,2,7,9,0,2,2,11,7,-1,-1,-1,-1}, {7,5,2,7,2,11,5,9,2,3,2,8,9,8,2,-1}, \
  {2,5,10,2,3,5,3,7,5,-1,-1,-1,-1,-1,-1,-1}, {8,2,0,8,5,2,8,7,5,10,2,5,-1,-1,-1,-1}, {9,0,1,5,10,3,5,3,7,3,10,2,-1,-1,-1,-1}, {9,8,2,9,2,1,8,7,2,10,2,5,7,5,2,-1}, \
  {1,3,5,3,7,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,8,7,0,7,1,1,7,5,-1,-1,-1,-1,-1,-1,-1}, {9,0,3,9,3,5,5,3,7,-1,-1,-1,-1,-1,-1,-1}, {9,8,7,5,9,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {5,8,4,5,10,8,10,11,8,-1,-1,-1,-1,-1,-1,-1}, {5,0,4,5,11,0,5,10,11,11,3,0,-1,-1,-1,-1}, {0,1,9,8,4,10,8,10,11,10,4,5,-1,-1,-1,-1}, {10,11,4,10,4,5,11,3,4,9,4,1,3,1,4,-1}, \
  {2,5,1,2,8,5,2,11,8,4,5,8,-1,-1,-1,-1}, {0,4,11,0,11,3,4,5,11,2,11,1,5,1,11,-1}, {0,2,5,0,5,9,2,11,5,4,5,8,11,8,5,-1}, {9,4,5,2,11,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {2,5,10,3,5,2,3,4,5,3,8,4,-1,-1,-1,-1}, {5,10,2,5,2,4,4,2,0,-1,-1,-1,-1,-1,-1,-1}, {3,10,2,3,5,10,3,8,5,4,5,8,0,1,9,-1}, {5,10,2,5,2,4,1,9,2,9,4,2,-1,-1,-1,-1}, \
  {8,4,5,8,5,3,3,5,1,-1,-1,-1,-1,-1,-1,-1}, {0,4,5,1,0,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {8,4,5,8,5,3,9,0,5,0,3,5,-1,-1,-1,-1}, {9,4,5,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {4,11,7,4,9,11,9,10,11,-1,-1,-1,-1,-1,-1,-1}, {0,8,3,4,9,7,9,11,7,9,10,11,-1,-1,-1,-1}, {1,10,11,1,11,4,1,4,0,7,4,11,-1,-1,-1,-1}, {3,1,4,3,4,8,1,10,4,7,4,11,10,11,4,-1}, \
  {4,11,7,9,11,4,9,2,11,9,1,2,-1,-1,-1,-1}, {9,7,4,9,11,7,9,1,11,2,11,1,0,8,3,-1}, {11,7,4,11,4,2,2,4,0,-1,-1,-1,-1,-1,-1,-1}, {11,7,4,11,4,2,8,3,4,3,2,4,-1,-1,-1,-1}, \
  {2,9,10,2,7,9,2,3,7,7,4,9,-1,-1,-1,-1}, {9,10,7,9,7,4,10,2,7,8,7,0,2,0,7,-1}, {3,7,10,3,10,2,7,4,10,1,10,0,4,0,10,-1}, {1,10,2,8,7,4,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {4,9,1,4,1,7,7,1,3,-1,-1,-1,-1,-1,-1,-1}, {4,9,1,4,1,7,0,8,1,8,7,1,-1,-1,-1,-1}, {4,0,3,7,4,3,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {4,8,7,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {9,10,8,10,11,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,0,9,3,9,11,11,9,10,-1,-1,-1,-1,-1,-1,-1}, {0,1,10,0,10,8,8,10,11,-1,-1,-1,-1,-1,-1,-1}, {3,1,10,11,3,10,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,2,11,1,11,9,9,11,8,-1,-1,-1,-1,-1,-1,-1}, {3,0,9,3,9,11,1,2,9,2,11,9,-1,-1,-1,-1}, {0,2,11,8,0,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {3,2,11,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {2,3,8,2,8,10,10,8,9,-1,-1,-1,-1,-1,-1,-1}, {9,10,2,0,9,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {2,3,8,2,8,10,0,1,8,1,10,8,-1,-1,-1,-1}, {1,10,2,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
  {1,3,8,9,1,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,9,1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {0,3,8,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, {-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1,-1}, \
}

__constant__ int8_t c_tri[256][16] = DGR_MC_TRI_TABLE;
const int8_t h_tri[256][16] = DGR_MC_TRI_TABLE;

// the two corners of edges 0..11, and each edge's owner: its lower endpoint (offset from the cube's voxel) and axis
__constant__ int8_t c_edge_corner[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6},
                                            {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
const int8_t h_edge_corner[12][2] = {{0, 1}, {1, 2}, {2, 3}, {3, 0}, {4, 5}, {5, 6},
                                     {6, 7}, {7, 4}, {0, 4}, {1, 5}, {2, 6}, {3, 7}};
__constant__ int8_t c_edge_owner[12][4] = {{0, 0, 0, 0}, {1, 0, 0, 1}, {0, 1, 0, 0}, {0, 0, 0, 1},
                                           {0, 0, 1, 0}, {1, 0, 1, 1}, {0, 1, 1, 0}, {0, 0, 1, 1},
                                           {0, 0, 0, 2}, {1, 0, 0, 2}, {1, 1, 0, 2}, {0, 1, 0, 2}};
__constant__ int8_t c_corner[8][3] = {{0, 0, 0}, {1, 0, 0}, {1, 1, 0}, {0, 1, 0},
                                      {0, 0, 1}, {1, 0, 1}, {1, 1, 1}, {0, 1, 1}};

__device__ __forceinline__ uint64_t unit_key(int x, int y, int z) {
  return (uint64_t)(uint32_t)(x + kCoordBias) | ((uint64_t)(uint32_t)(y + kCoordBias) << 21) |
         ((uint64_t)(uint32_t)(z + kCoordBias) << 42);
}

// camera model: intrinsics and rows 0..2 of a 4x4 (camera_pose for the touch pass, extrinsic for integration)
struct Cam {
  double fx, fy, cx, cy;
  double M[12];
};

// row r of M applied to (x, y, z): ((M0 x + M1 y) + M2 z) + M3
__device__ __forceinline__ double affine_row(const double* M, double x, double y, double z) {
  return __dadd_rn(__dadd_rn(__dadd_rn(__dmul_rn(M[0], x), __dmul_rn(M[1], y)), __dmul_rn(M[2], z)), M[3]);
}

// ---------------------------------------------------------------------------------------
// touch / allocate
// ---------------------------------------------------------------------------------------
// Candidate row s * side^3 + (ox side + oy) side + oz of sample s (row-major over the strided grid): the unit
// lo + o when it lies within [lo, hi] on every axis and the sample has depth, else the sentinel (kSentinel)^3.
__global__ void __launch_bounds__(kThreads)
touch_kernel(const float* __restrict__ depth, int W, int stride, int Ws, int64_t n_samples, Cam cam, double L,
             double trunc, int side, int32_t* __restrict__ cand, int32_t* __restrict__ counts,
             dgr_keyspec_t* __restrict__ spec) {
  const int64_t s = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (s == 0) {
    dgr_keyspec_t k{};
    k.ncols = 3;
    for (int a = 0; a < 3; ++a) {
      k.lo[a] = -kCoordBias;
      k.shift[a] = 21 * a;
      k.bits[a] = 21;
    }
    *spec = k;
  }
  if (s >= n_samples) return;
  const int i = (int)(s / Ws) * stride, j = (int)(s % Ws) * stride;
  const float df = depth[(int64_t)i * W + j];
  int lo[3] = {0, 0, 0}, hi[3] = {-1, -1, -1};
  if (df > 0.f) {
    const double d = (double)df;
    const double x = __ddiv_rn(__dmul_rn(__dsub_rn((double)j, cam.cx), d), cam.fx);
    const double y = __ddiv_rn(__dmul_rn(__dsub_rn((double)i, cam.cy), d), cam.fy);
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const double p = affine_row(cam.M + 4 * a, x, y, d);
      lo[a] = (int)floor(__ddiv_rn(__dsub_rn(p, trunc), L));
      hi[a] = (int)floor(__ddiv_rn(__dadd_rn(p, trunc), L));
    }
  }
  const int n_c = side * side * side;
  bool bad = false;
  for (int c = 0; c < n_c; ++c) {
    const int o[3] = {c / (side * side), (c / side) % side, c % side};
    int u[3] = {kSentinel, kSentinel, kSentinel};
    bool in = true, range = true;
#pragma unroll
    for (int a = 0; a < 3; ++a) {
      const int q = lo[a] + o[a];
      in = in && q <= hi[a];
      range = range && q >= DGR_TSDF_COORD_MIN && q <= DGR_TSDF_COORD_MAX;
    }
    if (in && range) {
#pragma unroll
      for (int a = 0; a < 3; ++a) u[a] = lo[a] + o[a];
    }
    bad = bad || (in && !range);
    int32_t* dst = cand + 3 * (s * n_c + c);
    dst[0] = u[0];
    dst[1] = u[1];
    dst[2] = u[2];
  }
  if (bad) counts[2] = 1;
}

// Unique candidate r (first-occurrence rank, r < m): its slot in the volume table (tslot), or -1 and flag = 1 when
// it is new; the sentinel keeps tslot = -1, flag = 0.  Per-256 block flag counts go to blk.
__global__ void __launch_bounds__(256)
touch_lookup_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ sel,
                    const int32_t* __restrict__ n_unique, int64_t n_max, const uint64_t* __restrict__ keys,
                    const int32_t* __restrict__ vals, uint64_t mask, int32_t* __restrict__ tslot,
                    int32_t* __restrict__ flag, int32_t* __restrict__ blk) {
  const int m = *n_unique;
  const int64_t r = (int64_t)blockIdx.x * 256 + threadIdx.x;
  int f = 0;
  if (r < m) {
    const int32_t* c = cand + 3 * (int64_t)sel[r];
    int32_t slot = -1;
    if (c[0] != kSentinel) {
      slot = dgr_hash_lookup(keys, vals, mask, unit_key(c[0], c[1], c[2]));
      f = slot < 0;
    }
    tslot[r] = slot;
  }
  if (r < n_max) flag[r] = f;
  int tot;
  dgr_block_exclusive_scan<256>(f, &tot);
  if (threadIdx.x == 0) blk[blockIdx.x] = tot;
}

// New unit q (in rank order) takes slot n_total + q: inserted into the volume table, its key written.
__global__ void __launch_bounds__(256)
touch_insert_kernel(const int32_t* __restrict__ cand, const int32_t* __restrict__ sel,
                    const int32_t* __restrict__ sel_new, const int32_t* __restrict__ n_new_p, int n_total,
                    uint64_t* __restrict__ keys, int32_t* __restrict__ vals, uint64_t mask,
                    int32_t* __restrict__ unit_keys, int32_t* __restrict__ tslot) {
  const int n_new = *n_new_p;
  const int q = blockIdx.x * 256 + threadIdx.x;
  if (q >= n_new) return;
  const int r = sel_new[q];
  const int32_t* c = cand + 3 * (int64_t)sel[r];
  const int slot = n_total + q;
  const uint32_t h = dgr_hash_insert(keys, mask, unit_key(c[0], c[1], c[2]));
  vals[h] = slot;
  unit_keys[3 * (int64_t)slot] = c[0];
  unit_keys[3 * (int64_t)slot + 1] = c[1];
  unit_keys[3 * (int64_t)slot + 2] = c[2];
  tslot[r] = slot;
}

// touched[] = the slots of the unique candidates in rank order without the sentinel; counts = (n_touched, n_total)
__global__ void __launch_bounds__(256)
touch_compact_kernel(const int32_t* __restrict__ tslot, const int32_t* __restrict__ n_unique,
                     const uint64_t* __restrict__ dkeys, const int32_t* __restrict__ dvals, uint64_t dmask,
                     const int32_t* __restrict__ n_new_p, int n_total, int32_t* __restrict__ touched,
                     int32_t* __restrict__ counts) {
  const int m = *n_unique;
  const int sent = dgr_hash_lookup(dkeys, dvals, dmask, unit_key(kSentinel, kSentinel, kSentinel));
  const int r = blockIdx.x * 256 + threadIdx.x;
  if (r == 0) {
    counts[0] = m - (sent >= 0);
    counts[1] = n_total + *n_new_p;
  }
  if (r >= m || r == sent) return;
  touched[r - (sent >= 0 && sent < r)] = tslot[r];
}

__global__ void rehash_kernel(const int32_t* __restrict__ unit_keys, int n, uint64_t* __restrict__ keys,
                              int32_t* __restrict__ vals, uint64_t mask) {
  const int s = blockIdx.x * blockDim.x + threadIdx.x;
  if (s >= n) return;
  const int32_t* c = unit_keys + 3 * (int64_t)s;
  vals[dgr_hash_insert(keys, mask, unit_key(c[0], c[1], c[2]))] = s;
}

// ---------------------------------------------------------------------------------------
// integrate
// ---------------------------------------------------------------------------------------
__global__ void __launch_bounds__(kThreads)
integrate_kernel(const float* __restrict__ depth, const uint8_t* __restrict__ color, int W, int H, Cam cam, double vl,
                 double L, float trunc32, float inv32, const int32_t* __restrict__ unit_keys,
                 const int32_t* __restrict__ touched, float* __restrict__ tsdf, float* __restrict__ weight,
                 float* __restrict__ rgb) {
  const int slot = touched[blockIdx.x];
  const double bx = __dmul_rn((double)unit_keys[3 * (int64_t)slot], L);
  const double by = __dmul_rn((double)unit_keys[3 * (int64_t)slot + 1], L);
  const double bz = __dmul_rn((double)unit_keys[3 * (int64_t)slot + 2], L);
  const double umax = __dsub_rn((double)W, 0.0001), vmax = __dsub_rn((double)H, 0.0001);
  float* ts = tsdf + (int64_t)slot * kVox;
  float* wt = weight + (int64_t)slot * kVox;
#pragma unroll 2
  for (int k = 0; k < kPerThread; ++k) {
    const int v = threadIdx.x + kThreads * k;
    const double X = __dadd_rn(bx, __dmul_rn((double)(v >> 8) + 0.5, vl));
    const double Y = __dadd_rn(by, __dmul_rn((double)((v >> 4) & 15) + 0.5, vl));
    const double Z = __dadd_rn(bz, __dmul_rn((double)(v & 15) + 0.5, vl));
    const double cz = affine_row(cam.M + 8, X, Y, Z);
    if (!(cz > 0.0)) continue;
    const double cx = affine_row(cam.M, X, Y, Z), cy = affine_row(cam.M + 4, X, Y, Z);
    const double uf = __dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(cx, cam.fx), cz), cam.cx), 0.5);
    const double vf = __dadd_rn(__dadd_rn(__ddiv_rn(__dmul_rn(cy, cam.fy), cz), cam.cy), 0.5);
    if (!(uf >= 0.0001 && uf < umax && vf >= 0.0001 && vf < vmax)) continue;
    const int u = (int)uf, r = (int)vf;
    const float d = depth[(int64_t)r * W + u];
    if (!(d > 0.f)) continue;
    const double a = __ddiv_rn(__dsub_rn((double)u, cam.cx), cam.fx);
    const double b = __ddiv_rn(__dsub_rn((double)r, cam.cy), cam.fy);
    const float mult = __double2float_rn(__dsqrt_rn(__dadd_rn(__dadd_rn(1.0, __dmul_rn(a, a)), __dmul_rn(b, b))));
    const float sdf = __fmul_rn(__double2float_rn(__dsub_rn((double)d, cz)), mult);
    if (!(sdf > -trunc32)) continue;
    const float tn = fminf(1.f, __fmul_rn(sdf, inv32));
    const float w0 = wt[v], w1 = __fadd_rn(w0, 1.f);
    ts[v] = __fdiv_rn(__fadd_rn(__fmul_rn(ts[v], w0), tn), w1);
    if (rgb != nullptr) {
      const uint8_t* px = color + 3 * ((int64_t)r * W + u);
#pragma unroll
      for (int c = 0; c < 3; ++c) {
        float* cc = rgb + ((int64_t)slot * 3 + c) * kVox + v;
        *cc = __fdiv_rn(__fadd_rn(__fmul_rn(*cc, w0), (float)px[c]), w1);
      }
    }
    wt[v] = w1;
  }
}

// ---------------------------------------------------------------------------------------
// extract
// ---------------------------------------------------------------------------------------
// Neighbour b = 4 dx + 2 dy + dz (d* in {0, 1}) of a local coordinate in [0, 16] per axis, and the voxel index in it
__device__ __forceinline__ int halo_nb(int x, int y, int z) { return ((x >> 4) << 2) | ((y >> 4) << 1) | (z >> 4); }
__device__ __forceinline__ int halo_lv(int x, int y, int z) { return ((x & 15) << 8) | ((y & 15) << 4) | (z & 15); }

__device__ __forceinline__ int tri_count(int idx) {
  int n = 0;
  while (n < 5 && c_tri[idx][3 * n] >= 0) ++n;
  return n;
}

// Rank of vertex (voxel lv, axis) among the unit's vertices ordered by (voxel, axis)
__device__ __forceinline__ int vertex_rank(const uint32_t* __restrict__ mask, const int32_t* __restrict__ wpre, int lv,
                                           int axis) {
  const int w = lv >> 5, bit = lv & 31;
  const uint32_t below = (1u << bit) - 1u;
  int r = wpre[w];
#pragma unroll
  for (int a = 0; a < 3; ++a) {
    const uint32_t m = mask[a * kMaskWords + w];
    r += __popc(m & below) + (a < axis ? (int)((m >> bit) & 1u) : 0);
  }
  return r;
}

struct ExtractWs {
  int32_t* nb;        // [n][8] slots of the unit and its +1 neighbours (-1: missing)
  uint8_t* cube;      // [n][4096] cube index of kept cubes, else 0
  uint32_t* mask;     // [n][3][128] owned-edge vertex bits
  int32_t* wpre;      // [n][128] vertices before each 32-voxel word
  int32_t* vcnt;      // [n + 1] vertices per unit, then their exclusive scan
  int32_t* tcnt;      // [n + 1] triangles per unit, then their exclusive scan
};

ExtractWs carve_extract(void* base, int64_t n, int64_t* words) {
  DgrCarver cv(base);
  ExtractWs w;
  w.nb = cv.take<int32_t>(n * 8);
  w.cube = cv.take<uint8_t>(n * kVox);
  w.mask = cv.take<uint32_t>(n * 3 * kMaskWords);
  w.wpre = cv.take<int32_t>(n * kMaskWords);
  w.vcnt = cv.take<int32_t>(n + 1);
  w.tcnt = cv.take<int32_t>(n + 1);
  if (words != nullptr) *words = cv.words;
  return w;
}

__global__ void __launch_bounds__(kThreads)
classify_kernel(const int32_t* __restrict__ unit_keys, const uint64_t* __restrict__ keys,
                const int32_t* __restrict__ vals, uint64_t mask, const float* __restrict__ tsdf,
                const float* __restrict__ weight, ExtractWs w) {
  __shared__ float f_s[kHaloN];
  __shared__ float w_s[kHaloN];
  __shared__ int nb_s[8];
  const int slot = blockIdx.x;
  if (threadIdx.x < 8) {
    const int b = threadIdx.x;
    const int32_t* c = unit_keys + 3 * (int64_t)slot;
    const int s = b == 0 ? slot : dgr_hash_lookup(keys, vals, mask, unit_key(c[0] + (b >> 2), c[1] + ((b >> 1) & 1),
                                                                            c[2] + (b & 1)));
    nb_s[b] = s;
    w.nb[(int64_t)slot * 8 + b] = s;
  }
  __syncthreads();
  for (int h = threadIdx.x; h < kHaloN; h += kThreads) {
    const int x = h / (kHalo * kHalo), y = (h / kHalo) % kHalo, z = h % kHalo;
    const int s = nb_s[halo_nb(x, y, z)];
    const int64_t g = (int64_t)s * kVox + halo_lv(x, y, z);
    f_s[h] = s >= 0 ? tsdf[g] : 0.f;
    w_s[h] = s >= 0 ? weight[g] : 0.f;
  }
  __syncthreads();
  int ntri = 0;
  for (int k = 0; k < kPerThread; ++k) {
    const int v = threadIdx.x + kThreads * k;
    const int x = v >> 8, y = (v >> 4) & 15, z = v & 15;
    int idx = 0;
    bool kept = true;
#pragma unroll
    for (int c = 0; c < 8; ++c) {
      const int h = ((x + c_corner[c][0]) * kHalo + (y + c_corner[c][1])) * kHalo + (z + c_corner[c][2]);
      kept = kept && w_s[h] != 0.f;
      idx |= (f_s[h] < 0.f) << c;
    }
    kept = kept && idx != 0 && idx != 255;
    w.cube[(int64_t)slot * kVox + v] = kept ? (uint8_t)idx : 0;
    if (!kept) continue;
    ntri += tri_count(idx);
    for (int e = 0; e < 12; ++e) {
      if (!(((idx >> c_edge_corner[e][0]) ^ (idx >> c_edge_corner[e][1])) & 1)) continue;
      const int ox = x + c_edge_owner[e][0], oy = y + c_edge_owner[e][1], oz = z + c_edge_owner[e][2];
      const int s = nb_s[halo_nb(ox, oy, oz)];
      const int lv = halo_lv(ox, oy, oz);
      atomicOr(w.mask + ((int64_t)s * 3 + c_edge_owner[e][3]) * kMaskWords + (lv >> 5), 1u << (lv & 31));
    }
  }
  int tot;
  dgr_block_exclusive_scan<kThreads>(ntri, &tot);
  if (threadIdx.x == 0) w.tcnt[slot] = tot;
}

__global__ void __launch_bounds__(kMaskWords) vertex_count_kernel(ExtractWs w) {
  const int slot = blockIdx.x, t = threadIdx.x;
  const uint32_t* m = w.mask + (int64_t)slot * 3 * kMaskWords;
  const int c = __popc(m[t]) + __popc(m[kMaskWords + t]) + __popc(m[2 * kMaskWords + t]);
  int tot;
  w.wpre[(int64_t)slot * kMaskWords + t] = dgr_block_exclusive_scan<kMaskWords>(c, &tot);
  if (t == 0) w.vcnt[slot] = tot;
}

__global__ void totals_kernel(const int32_t* __restrict__ vcnt, const int32_t* __restrict__ tcnt, int n,
                              int32_t* __restrict__ totals) {
  totals[0] = vcnt[n];
  totals[1] = tcnt[n];
}

__global__ void __launch_bounds__(kThreads)
write_vertices_kernel(const int32_t* __restrict__ unit_keys, const float* __restrict__ tsdf,
                      const float* __restrict__ rgb, double vl, ExtractWs w, double* __restrict__ verts,
                      double* __restrict__ colors) {
  const int slot = blockIdx.x;
  const int32_t* nb = w.nb + (int64_t)slot * 8;
  const uint32_t* m = w.mask + (int64_t)slot * 3 * kMaskWords;
  const int32_t* wpre = w.wpre + (int64_t)slot * kMaskWords;
  const int base = w.vcnt[slot];
  const int g0[3] = {unit_keys[3 * (int64_t)slot] * kRes, unit_keys[3 * (int64_t)slot + 1] * kRes,
                     unit_keys[3 * (int64_t)slot + 2] * kRes};
  for (int k = 0; k < kPerThread; ++k) {
    const int v = threadIdx.x + kThreads * k;
    const int l[3] = {v >> 8, (v >> 4) & 15, v & 15};
    for (int a = 0; a < 3; ++a) {
      if (!((m[a * kMaskWords + (v >> 5)] >> (v & 31)) & 1u)) continue;
      const int id = base + vertex_rank(m, wpre, v, a);
      int l1[3] = {l[0], l[1], l[2]};
      ++l1[a];
      const int s1 = nb[halo_nb(l1[0], l1[1], l1[2])], v1 = halo_lv(l1[0], l1[1], l1[2]);
      const double a0 = fabs((double)tsdf[(int64_t)slot * kVox + v]);
      const double a1 = fabs((double)tsdf[(int64_t)s1 * kVox + v1]);
      const double den = __dadd_rn(a0, a1);
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        double p = __dmul_rn(__dadd_rn((double)(g0[q] + l[q]), 0.5), vl);
        if (q == a) p = __dadd_rn(p, __ddiv_rn(__dmul_rn(a0, vl), den));
        verts[3 * (int64_t)id + q] = p;
      }
      if (colors != nullptr) {
#pragma unroll
        for (int c = 0; c < 3; ++c) {
          const double c0 = (double)rgb[((int64_t)slot * 3 + c) * kVox + v];
          const double c1 = (double)rgb[((int64_t)s1 * 3 + c) * kVox + v1];
          colors[3 * (int64_t)id + c] =
              __ddiv_rn(__ddiv_rn(__dadd_rn(__dmul_rn(a1, c0), __dmul_rn(a0, c1)), den), 255.0);
        }
      }
    }
  }
}

__global__ void __launch_bounds__(kThreads) write_triangles_kernel(ExtractWs w, int32_t* __restrict__ tris) {
  const int slot = blockIdx.x;
  __shared__ int nb_s[8];
  if (threadIdx.x < 8) nb_s[threadIdx.x] = w.nb[(int64_t)slot * 8 + threadIdx.x];
  __syncthreads();
  int run = w.tcnt[slot];
  for (int k = 0; k < kPerThread; ++k) {
    const int v = kThreads * k + threadIdx.x;          // 256 consecutive voxels per step, in voxel order
    const int idx = w.cube[(int64_t)slot * kVox + v];
    const int n = idx != 0 ? tri_count(idx) : 0;
    int tot;
    int pos = run + dgr_block_exclusive_scan<kThreads>(n, &tot);
    const int x = v >> 8, y = (v >> 4) & 15, z = v & 15;
    for (int t = 0; t < n; ++t) {
      int id[3];
#pragma unroll
      for (int q = 0; q < 3; ++q) {
        const int e = c_tri[idx][3 * t + q];
        const int ox = x + c_edge_owner[e][0], oy = y + c_edge_owner[e][1], oz = z + c_edge_owner[e][2];
        const int s = nb_s[halo_nb(ox, oy, oz)];
        id[q] = w.vcnt[s] + vertex_rank(w.mask + (int64_t)s * 3 * kMaskWords, w.wpre + (int64_t)s * kMaskWords,
                                        halo_lv(ox, oy, oz), c_edge_owner[e][3]);
      }
      int32_t* dst = tris + 3 * (int64_t)pos;
      dst[0] = id[0];                                   // open3d's winding (e[i], e[i+2], e[i+1])
      dst[1] = id[2];
      dst[2] = id[1];
      ++pos;
    }
    run += tot;
    __syncthreads();                                   // the scan's warp totals are reused by the next step
  }
}

// ---------------------------------------------------------------------------------------
// ray cast (oracle/tsdf_raycast.py states the contract)
// ---------------------------------------------------------------------------------------
constexpr int kRayBx = 8, kRayBy = 16;         // 128 threads; a warp covers an 8 x 4 pixel tile

// Slot of the unit holding lattice voxel g (fp64 integers), its local index in lv; -1 when the unit is missing or
// outside the key range.  U receives the unit coordinates (fp64) either way.
__device__ __forceinline__ int ray_unit(const double g[3], const uint64_t* __restrict__ keys,
                                        const int32_t* __restrict__ vals, uint64_t mask, bool have_table, double U[3],
                                        int& lv) {
  bool in = have_table;
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    U[k] = floor(__dmul_rn(g[k], 0.0625));
    in = in && U[k] >= (double)DGR_TSDF_COORD_MIN && U[k] <= (double)DGR_TSDF_COORD_MAX;
  }
  if (!in) return -1;
  const int ux = (int)U[0], uy = (int)U[1], uz = (int)U[2];
  lv = (((int)g[0] - kRes * ux) * kRes + ((int)g[1] - kRes * uy)) * kRes + ((int)g[2] - kRes * uz);
  return dgr_hash_lookup(keys, vals, mask, unit_key(ux, uy, uz));
}

// Steps a ray of the launch may take: ceil(((2 s_max) depth_max) / voxel_length) + 1, where s_max is the largest
// world length per unit of t over the image.  s = |R (a, b, 1)| is convex in (a, b), so its maximum over the image
// lies at a corner pixel.  Every step advances t by at least (0.5 voxel_length) / s, so no ray needs more.
double raycast_max_steps(int W, int H, const double* intr, const double* M, double vl, double dmax) {
  double s_max = 0.0;
  for (int c = 0; c < 4; ++c) {
    const double a = ((double)((c & 1) ? W - 1 : 0) - intr[2]) / intr[0];
    const double b = ((double)((c & 2) ? H - 1 : 0) - intr[3]) / intr[1];
    double d[3];
    for (int k = 0; k < 3; ++k) d[k] = (M[4 * k] * a + M[4 * k + 1] * b) + M[4 * k + 2];
    const double s = sqrt((d[0] * d[0] + d[1] * d[1]) + d[2] * d[2]);
    s_max = s > s_max ? s : s_max;
  }
  return ceil(((2.0 * s_max) * dmax) / vl) + 1.0;
}

// One thread per pixel (u, v): march p(t) = C + t d from depth_min, sample the voxel holding p, stop at the first
// (known > 0, known <= 0) pair of consecutive known samples; a missing-unit jump breaks the pair, an unknown voxel
// does not.  Read-only on the volume; writes every output pixel.
__global__ void __launch_bounds__(kRayBx* kRayBy)
raycast_kernel(const uint64_t* __restrict__ keys, const int32_t* __restrict__ vals, uint64_t mask, bool have_table,
               const float* __restrict__ tsdf, const float* __restrict__ weight, const float* __restrict__ rgb, int W,
               int H, Cam cam, double vl, double trunc, double dmin, double dmax, double wthr, int max_steps,
               float* __restrict__ depth, float* __restrict__ intensity, float* __restrict__ colour) {
  const int u = blockIdx.x * kRayBx + threadIdx.x, v = blockIdx.y * kRayBy + threadIdx.y;
  if (u >= W || v >= H) return;
  const double a = __ddiv_rn(__dsub_rn((double)u, cam.cx), cam.fx);
  const double b = __ddiv_rn(__dsub_rn((double)v, cam.cy), cam.fy);
  double C[3], d[3];
#pragma unroll
  for (int k = 0; k < 3; ++k) {
    d[k] = __dadd_rn(__dadd_rn(__dmul_rn(cam.M[4 * k], a), __dmul_rn(cam.M[4 * k + 1], b)), cam.M[4 * k + 2]);
    C[k] = cam.M[4 * k + 3];
  }
  const double s = __dsqrt_rn(__dadd_rn(__dadd_rn(__dmul_rn(d[0], d[0]), __dmul_rn(d[1], d[1])), __dmul_rn(d[2], d[2])));
  const double dt_vox = __ddiv_rn(vl, s), dt_half = __ddiv_rn(__dmul_rn(0.5, vl), s);
  double t = dmin, tp = 0.0, t_hit = 0.0;
  float fp = 0.f;
  bool prev = false, hit = false;
  for (int n = 0; n < max_steps && t <= dmax; ++n) {    // the cap is the host's bound: it never cuts a ray short
    double g[3], U[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) g[k] = floor(__ddiv_rn(__dadd_rn(C[k], __dmul_rn(t, d[k])), vl));
    int lv = 0;
    const int slot = ray_unit(g, keys, vals, mask, have_table, U, lv);
    if (slot < 0) {                                    // missing unit: past its exit plane, plus half a voxel
      double te = CUDART_INF;
#pragma unroll
      for (int k = 0; k < 3; ++k) {
        if (d[k] == 0.0) continue;
        const double bnd = __dmul_rn(__dadd_rn(__dmul_rn(U[k], 16.0), d[k] > 0.0 ? 16.0 : 0.0), vl);
        const double tk = __ddiv_rn(__dsub_rn(bnd, C[k]), d[k]);
        te = tk < te ? tk : te;
      }
      t = __dadd_rn(te > t ? te : t, dt_half);
      prev = false;
      continue;
    }
    const int64_t at = (int64_t)slot * kVox + lv;
    const float w = weight[at];
    if (!((double)w >= wthr)) {                        // unknown voxel of an existing unit: one voxel on
      t = __dadd_rn(t, dt_vox);
      continue;
    }
    const float f = tsdf[at];
    if (prev && fp > 0.f && f <= 0.f) {
      t_hit = __dadd_rn(tp, __dmul_rn(__dsub_rn(t, tp), __ddiv_rn((double)fp, __dsub_rn((double)fp, (double)f))));
      hit = t_hit >= dmin && t_hit <= dmax;
      break;
    }
    prev = true;
    fp = f;
    tp = t;
    const double step = __dmul_rn((double)f, trunc);
    t = __dadd_rn(t, __ddiv_rn(step > vl ? step : vl, s));
  }
  const int64_t px = (int64_t)v * W + u;
  depth[px] = hit ? __double2float_rn(t_hit) : 0.f;
  if (intensity == nullptr && colour == nullptr) return;
  float c32[3] = {0.f, 0.f, 0.f};
  if (hit) {                                           // trilinear over the 8 voxels around p(t_hit) with weight > 0
    double q[3], g0[3], fr[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
      q[k] = __dsub_rn(__ddiv_rn(__dadd_rn(C[k], __dmul_rn(t_hit, d[k])), vl), 0.5);
      g0[k] = floor(q[k]);
      fr[k] = __dsub_rn(q[k], g0[k]);
    }
    double acc[3] = {0.0, 0.0, 0.0}, wsum = 0.0;
    for (int c = 0; c < 8; ++c) {
      const int o[3] = {c >> 2, (c >> 1) & 1, c & 1};
      double g[3], U[3];
#pragma unroll
      for (int k = 0; k < 3; ++k) g[k] = __dadd_rn(g0[k], (double)o[k]);
      int lv = 0;
      const int slot = ray_unit(g, keys, vals, mask, have_table, U, lv);
      const int64_t at = (int64_t)slot * kVox + lv;
      if (slot < 0 || !(weight[at] > 0.f)) continue;
      const double tw = __dmul_rn(__dmul_rn(o[0] ? fr[0] : __dsub_rn(1.0, fr[0]), o[1] ? fr[1] : __dsub_rn(1.0, fr[1])),
                                  o[2] ? fr[2] : __dsub_rn(1.0, fr[2]));
#pragma unroll
      for (int k = 0; k < 3; ++k)
        acc[k] = __dadd_rn(acc[k], __dmul_rn(tw, (double)rgb[((int64_t)slot * 3 + k) * kVox + lv]));
      wsum = __dadd_rn(wsum, tw);
    }
    if (wsum > 0.0) {
#pragma unroll
      for (int k = 0; k < 3; ++k) c32[k] = __double2float_rn(__ddiv_rn(acc[k], wsum));
    }
  }
  if (intensity != nullptr)                            // create_from_color_and_depth's intensity, fp32
    intensity[px] = __fdiv_rn(__fadd_rn(__fadd_rn(__fmul_rn(c32[0], 0.299f), __fmul_rn(c32[1], 0.587f)),
                                        __fmul_rn(c32[2], 0.114f)), 255.f);
  if (colour != nullptr) {
#pragma unroll
    for (int k = 0; k < 3; ++k) colour[3 * px + k] = __fdiv_rn(c32[k], 255.f);
  }
}

struct TouchWs {
  dgr_keyspec_t* spec;
  int32_t *cand, *sel, *inverse, *n_unique, *slot_ws, *scan_ws, *flag, *blk, *sel_new, *tslot, *dvals;
  uint64_t* dkeys;
};

int64_t side_of(double voxel_length, double sdf_trunc) {
  return (int64_t)floor(2.0 * sdf_trunc / (voxel_length * kRes)) + 2;
}

int64_t touch_candidates(int32_t width, int32_t height, int32_t stride, double voxel_length, double sdf_trunc) {
  const int64_t hs = (height + stride - 1) / stride, ws = (width + stride - 1) / stride, side = side_of(voxel_length,
                                                                                                         sdf_trunc);
  return hs * ws * side * side * side;
}

int64_t dedup_cap(int64_t n) {
  int64_t p = 1024;
  while (p < 2 * n) p <<= 1;
  return p;
}

TouchWs carve_touch(void* base, int64_t n, int64_t* words) {
  DgrCarver cv(base);
  TouchWs w;
  const int64_t cap = dedup_cap(n), nb = dgr_blocks(n, 256);
  w.spec = cv.take<dgr_keyspec_t>(1);
  w.cand = cv.take<int32_t>(3 * n);
  w.dkeys = cv.take<uint64_t>(cap);
  w.dvals = cv.take<int32_t>(cap);
  w.sel = cv.take<int32_t>(n);
  w.inverse = cv.take<int32_t>(n);
  w.n_unique = cv.take<int32_t>(2);
  w.slot_ws = cv.take<int32_t>(n);
  w.scan_ws = cv.take<int32_t>(dgr_scan_ws_elems(n));
  w.flag = cv.take<int32_t>(n);
  w.blk = cv.take<int32_t>(nb + 1);
  w.sel_new = cv.take<int32_t>(n);
  w.tslot = cv.take<int32_t>(n);
  if (words != nullptr) *words = cv.words;
  return w;
}

int32_t check_frame(int32_t width, int32_t height, const double* intr, double voxel_length, double sdf_trunc,
                    int32_t res) {
  DGR_ARG_CHECK(width >= 1 && height >= 1 && (int64_t)width * height < INT_MAX, "image size out of range");
  DGR_ARG_CHECK(res == kRes, "volume_unit_resolution must be 16 (DGR_TSDF_RES)");
  DGR_ARG_CHECK(voxel_length > 0 && voxel_length < 1e6, "voxel_length must be positive");
  DGR_ARG_CHECK(sdf_trunc > 0 && sdf_trunc < 1e6, "sdf_trunc must be positive");
  DGR_ARG_CHECK(intr != nullptr && intr[0] > 0 && intr[1] > 0, "focal lengths must be positive");
  return DGR_OK;
}

Cam make_cam(const double* intr, const double* M) {
  Cam c;
  c.fx = intr[0];
  c.fy = intr[1];
  c.cx = intr[2];
  c.cy = intr[3];
  for (int i = 0; i < 12; ++i) c.M[i] = M[i];
  return c;
}

}  // namespace

extern "C" {

int32_t dgr_tsdf_touch_ws_elems(int32_t width, int32_t height, int32_t stride, double voxel_length, double sdf_trunc,
                                int64_t* n_cand, int64_t* n_elems) {
  DGR_ARG_CHECK(n_cand != nullptr && n_elems != nullptr, "null output");
  DGR_ARG_CHECK(width >= 1 && height >= 1 && stride >= 1, "image size and stride must be positive");
  DGR_ARG_CHECK(voxel_length > 0 && sdf_trunc > 0, "voxel_length and sdf_trunc must be positive");
  const int64_t n = touch_candidates(width, height, stride, voxel_length, sdf_trunc);
  DGR_ARG_CHECK(n < (int64_t)INT_MAX / 4, "too many candidate units per frame");
  *n_cand = n;
  carve_touch(nullptr, n, n_elems);
  return DGR_OK;
}

int32_t dgr_tsdf_touch(const float* depth, int32_t width, int32_t height, const double* intr, const double* pose,
                       double voxel_length, double sdf_trunc, int32_t res, int32_t stride, uint64_t* table_keys,
                       int32_t* table_vals, int64_t table_cap, int32_t* unit_keys, int64_t unit_cap, int32_t n_total,
                       int32_t* touched, int32_t* counts, void* ws, void* stream) {
  if (int32_t e = check_frame(width, height, intr, voxel_length, sdf_trunc, res)) return e;
  DGR_ARG_CHECK(stride >= 1, "depth_sampling_stride must be >= 1");
  DGR_ARG_CHECK(pose != nullptr && depth != nullptr && touched != nullptr && counts != nullptr && ws != nullptr,
                "null argument");
  const int64_t n = touch_candidates(width, height, stride, voxel_length, sdf_trunc);
  DGR_ARG_CHECK(n < (int64_t)INT_MAX / 4, "too many candidate units per frame");
  DGR_ARG_CHECK(n_total >= 0 && unit_cap >= (int64_t)n_total + n, "unit_keys must hold n_total + the candidates");
  DGR_ARG_CHECK(table_cap > 0 && (table_cap & (table_cap - 1)) == 0 && table_cap >= 2 * ((int64_t)n_total + n),
                "table capacity: a power of two >= 2 (n_total + candidates)");
  cudaStream_t st = (cudaStream_t)stream;
  TouchWs w = carve_touch(ws, n, nullptr);
  const int64_t dcap = dedup_cap(n), nb = dgr_blocks(n, 256);
  const int Ws = (width + stride - 1) / stride, Hs = (height + stride - 1) / stride;
  const int side = (int)side_of(voxel_length, sdf_trunc);
  DGR_CUDA_CHECK(cudaMemsetAsync(counts, 0, 3 * sizeof(int32_t), st));
  touch_kernel<<<dgr_blocks((int64_t)Ws * Hs, kThreads), kThreads, 0, st>>>(
      depth, width, stride, Ws, (int64_t)Ws * Hs, make_cam(intr, pose), voxel_length * kRes, sdf_trunc, side, w.cand,
      counts, w.spec);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  if (int32_t e = dgr_hash_clear(w.dkeys, w.dvals, dcap, stream)) return e;
  if (int32_t e = dgr_unique_first(w.cand, n, 3, w.spec, w.dkeys, w.dvals, dcap, w.sel, w.inverse, w.n_unique,
                                   w.slot_ws, w.scan_ws, stream))
    return e;
  touch_lookup_kernel<<<(unsigned)nb, 256, 0, st>>>(w.cand, w.sel, w.n_unique, n, table_keys, table_vals,
                                                   (uint64_t)table_cap - 1, w.tslot, w.flag, w.blk);
  dgr_scan_counts(w.blk, nb, st);
  dgr_select_first(w.flag, w.blk, n, n, 0, w.sel_new, nullptr, st);
  touch_insert_kernel<<<(unsigned)nb, 256, 0, st>>>(w.cand, w.sel, w.sel_new, w.blk + nb, n_total, table_keys,
                                                   table_vals, (uint64_t)table_cap - 1, unit_keys, w.tslot);
  touch_compact_kernel<<<(unsigned)nb, 256, 0, st>>>(w.tslot, w.n_unique, w.dkeys, w.dvals, (uint64_t)dcap - 1,
                                                    w.blk + nb, n_total, touched, counts);
  dgr_note_launches(5);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_tsdf_rehash(const int32_t* unit_keys, int32_t n_total, uint64_t* table_keys, int32_t* table_vals,
                        int64_t table_cap, void* stream) {
  DGR_ARG_CHECK(table_cap > 0 && (table_cap & (table_cap - 1)) == 0 && table_cap >= 2 * (int64_t)n_total,
                "table capacity: a power of two >= 2 n_total");
  if (int32_t e = dgr_hash_clear(table_keys, table_vals, table_cap, stream)) return e;
  if (n_total > 0) {
    rehash_kernel<<<dgr_blocks(n_total, 256), 256, 0, (cudaStream_t)stream>>>(unit_keys, n_total, table_keys,
                                                                             table_vals, (uint64_t)table_cap - 1);
    dgr_note_launches(1);
    DGR_LAUNCH_CHECK();
  }
  return DGR_OK;
}

int32_t dgr_tsdf_integrate(const float* depth, const uint8_t* color, int32_t width, int32_t height, const double* intr,
                           const double* extrinsic, double voxel_length, double sdf_trunc, int32_t res,
                           const int32_t* unit_keys, const int32_t* touched, int32_t n_touched, float* tsdf,
                           float* weight, float* rgb, int64_t slab_units, void* stream) {
  if (int32_t e = check_frame(width, height, intr, voxel_length, sdf_trunc, res)) return e;
  DGR_ARG_CHECK(extrinsic != nullptr && depth != nullptr, "null argument");
  DGR_ARG_CHECK((rgb == nullptr) == (color == nullptr), "colour image and colour slab go together");
  DGR_ARG_CHECK(n_touched >= 0 && n_touched <= slab_units, "more touched units than slab units");
  if (n_touched == 0) return DGR_OK;
  const float trunc32 = (float)sdf_trunc, inv32 = (float)(1.0 / sdf_trunc);
  integrate_kernel<<<n_touched, kThreads, 0, (cudaStream_t)stream>>>(
      depth, color, width, height, make_cam(intr, extrinsic), voxel_length, voxel_length * kRes, trunc32, inv32,
      unit_keys, touched, tsdf, weight, rgb);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_tsdf_extract_ws_elems(int64_t n_units, int64_t* n_elems) {
  DGR_ARG_CHECK(n_elems != nullptr && n_units >= 0, "bad arguments");
  carve_extract(nullptr, n_units, n_elems);
  return DGR_OK;
}

int32_t dgr_tsdf_extract_count(const int32_t* unit_keys, int32_t n_units, const uint64_t* table_keys,
                               const int32_t* table_vals, int64_t table_cap, const float* tsdf, const float* weight,
                               int32_t res, void* ws, int32_t* totals, void* stream) {
  DGR_ARG_CHECK(res == kRes, "volume_unit_resolution must be 16 (DGR_TSDF_RES)");
  DGR_ARG_CHECK(n_units >= 0 && totals != nullptr, "bad arguments");
  DGR_ARG_CHECK(table_cap > 0 && (table_cap & (table_cap - 1)) == 0, "table capacity must be a power of two");
  cudaStream_t st = (cudaStream_t)stream;
  if (n_units == 0) {
    DGR_CUDA_CHECK(cudaMemsetAsync(totals, 0, 2 * sizeof(int32_t), st));
    return DGR_OK;
  }
  ExtractWs w = carve_extract(ws, n_units, nullptr);
  DGR_CUDA_CHECK(cudaMemsetAsync(w.mask, 0, (size_t)n_units * 3 * kMaskWords * sizeof(uint32_t), st));
  classify_kernel<<<n_units, kThreads, 0, st>>>(unit_keys, table_keys, table_vals, (uint64_t)table_cap - 1, tsdf,
                                                weight, w);
  vertex_count_kernel<<<n_units, kMaskWords, 0, st>>>(w);
  dgr_scan_counts(w.vcnt, n_units, st);
  dgr_scan_counts(w.tcnt, n_units, st);
  totals_kernel<<<1, 1, 0, st>>>(w.vcnt, w.tcnt, n_units, totals);
  dgr_note_launches(5);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_tsdf_extract_write(const int32_t* unit_keys, int32_t n_units, const float* tsdf, const float* rgb,
                               double voxel_length, const void* ws, double* vertices, double* colors,
                               int32_t* triangles, void* stream) {
  DGR_ARG_CHECK(n_units >= 0 && voxel_length > 0, "bad arguments");
  DGR_ARG_CHECK((rgb == nullptr) == (colors == nullptr), "colour slab and colour output go together");
  if (n_units == 0) return DGR_OK;
  cudaStream_t st = (cudaStream_t)stream;
  ExtractWs w = carve_extract(const_cast<void*>(ws), n_units, nullptr);
  write_vertices_kernel<<<n_units, kThreads, 0, st>>>(unit_keys, tsdf, rgb, voxel_length, w, vertices, colors);
  write_triangles_kernel<<<n_units, kThreads, 0, st>>>(w, triangles);
  dgr_note_launches(2);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_tsdf_raycast(const uint64_t* table_keys, const int32_t* table_vals, int64_t table_cap, const float* tsdf,
                         const float* weight, const float* rgb, int32_t width, int32_t height, const double* intr,
                         const double* pose, double voxel_length, double sdf_trunc, int32_t res, double depth_min,
                         double depth_max, double weight_threshold, float* depth, float* intensity, float* colour,
                         void* stream) {
  if (int32_t e = check_frame(width, height, intr, voxel_length, sdf_trunc, res)) return e;
  DGR_ARG_CHECK(isfinite(intr[0]) && isfinite(intr[1]) && isfinite(intr[2]) && isfinite(intr[3]),
                "the intrinsic must be finite");
  DGR_ARG_CHECK(pose != nullptr && depth != nullptr, "null argument");
  bool finite = true;
  for (int i = 0; i < 12; ++i) finite = finite && isfinite(pose[i]);
  DGR_ARG_CHECK(finite, "the camera pose must be finite");
  DGR_ARG_CHECK(depth_min >= 0.0 && depth_min < depth_max && isfinite(depth_max), "need 0 <= depth_min < depth_max");
  DGR_ARG_CHECK(weight_threshold > 0.0 && isfinite(weight_threshold), "weight_threshold must be positive");
  DGR_ARG_CHECK(rgb != nullptr || table_cap == 0 || (intensity == nullptr && colour == nullptr),
                "intensity and colour need a colour (RGB8) volume");
  DGR_ARG_CHECK(table_cap == 0 || ((table_cap & (table_cap - 1)) == 0 && table_keys != nullptr &&
                                   table_vals != nullptr && tsdf != nullptr && weight != nullptr),
                "table capacity must be 0 (an empty volume) or a power of two with its table and slabs");
  const double max_steps = raycast_max_steps(width, height, intr, pose, voxel_length, depth_max);
  DGR_ARG_CHECK(max_steps <= (double)DGR_TSDF_RAYCAST_MAX_STEPS,
                "a ray could take more than DGR_TSDF_RAYCAST_MAX_STEPS steps: ceil(2 s_max depth_max / voxel_length) + 1, "
                "s_max the largest |R (a, b, 1)| over the image's corner pixels");
  const dim3 block(kRayBx, kRayBy), grid((width + kRayBx - 1) / kRayBx, (height + kRayBy - 1) / kRayBy);
  raycast_kernel<<<grid, block, 0, (cudaStream_t)stream>>>(
      table_keys, table_vals, (uint64_t)(table_cap > 0 ? table_cap - 1 : 0), table_cap > 0, tsdf, weight, rgb, width,
      height, make_cam(intr, pose), voxel_length, sdf_trunc, depth_min, depth_max, weight_threshold, (int)max_steps, depth,
      intensity, colour);
  dgr_note_launches(1);
  DGR_LAUNCH_CHECK();
  return DGR_OK;
}

int32_t dgr_tsdf_mc_tables(int32_t* edge_table, int32_t* tri_table) {
  DGR_ARG_CHECK(edge_table != nullptr && tri_table != nullptr, "null output");
  for (int i = 0; i < 256; ++i) {
    int m = 0;
    for (int e = 0; e < 12; ++e) m |= (((i >> h_edge_corner[e][0]) ^ (i >> h_edge_corner[e][1])) & 1) << e;
    edge_table[i] = m;
    for (int k = 0; k < 16; ++k) tri_table[16 * i + k] = h_tri[i][k];
  }
  return DGR_OK;
}

}  // extern "C"
