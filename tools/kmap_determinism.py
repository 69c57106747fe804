"""Build the same kernel map repeatedly on one cloud and compare every run with the first (and bucket kappa with its
mirror K-1-kappa, which holds the same number of pairs): a race shows up as a run that differs.
Usage: python tools/kmap_determinism.py [reps]"""
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np
import torch

from deepglobalregistration_b200.me.coords import CoordinateManager, CoordinateMapKey

reps = int(sys.argv[1]) if len(sys.argv) > 1 else 5
g = np.random.default_rng(3 + 9000)
c = np.unique(g.integers(-16, 16, size=(9000, 3)), axis=0)
c = c[g.permutation(len(c))]
coords = np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)
ct = torch.from_numpy(coords).cuda().contiguous()
ok = True
first = None
for r in range(reps):
  man = CoordinateManager(ct, assume_unique=True)
  _, km = man.kernel_map(CoordinateMapKey(1), 1, 3)
  run = (km.kofs_host.copy(), km.in_idx[:km.n_pairs].cpu().numpy(), km.out_idx[:km.n_pairs].cpu().numpy(),
         km.tile_k[:km.n_tiles].cpu().numpy(), km.tile_start[:km.n_tiles].cpu().numpy())
  counts = np.diff(run[0])
  sym = bool(np.array_equal(counts, counts[::-1]))
  same = first is None or all(np.array_equal(a, b) for a, b in zip(run, first))
  print(f'rep {r}: P {run[0][-1]} equal to run 0 {same} mirror-symmetric {sym}', flush=True)
  first = first or run
  ok &= same and sym
print('DETERMINISM', 'PASS' if ok else 'FAIL')
