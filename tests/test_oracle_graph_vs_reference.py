"""The oracle's ResUNetBN2C restatement (oracle/resunet.py) against the reference's OWN model code:
model/resunet.py + model/residual_block.py + model/common.py of the reference, run unmodified on the CPU
over oracle/me_cpu.py (a MinkowskiEngine-shaped module backed by oracle/sparse_ops.py), recorded in
tests/golden/reference_cpu.npz by tests/golden/make_golden_reference_cpu.py.  Same sparse operators on both
sides, so this isolates - and pins - the GRAPH: layer order, strides, transposed-convolution pairing, skip
concatenation order, norm placement, final bias and normalisation."""
import os

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle.resunet import resunet_forward


@pytest.fixture(scope='module')
def ref_outputs():
  return np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'reference_cpu.npz'))


def _cloud(seed, n, D, extent):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-extent, extent, size=(n, D)), axis=0)
  return np.concatenate([np.zeros((len(c), 1), np.int64), c], 1).astype(np.int32)


# cases in the order tests/golden/make_golden_reference_cpu.py recorded them (key graph_<index>)
CASES = [
    (3, 1, 32, 7, True, 600, 7),        # FCGF, 3DMatch setting (scripts/train_3dmatch.sh:19)
    (3, 1, 32, 5, True, 500, 9),        # FCGF, KITTI setting
    (6, 1, 1, 3, False, 300, 2),        # inlier network, 'ones' features
    (6, 6, 1, 3, False, 250, 2),        # inlier network, 'coords' features
]


@pytest.mark.parametrize('D,cin,cout,k1,normalize,n,extent', CASES)
def test_reference_graph_equals_oracle_restatement(ref_outputs, D, cin, cout, k1, normalize, n, extent):
  sd = syn.resunet_state_dict(D + k1, cin, cout, k1, D)
  g = torch.Generator().manual_seed(1)
  for k in sd:                                  # non-trivial BN statistics so a misplaced norm shows
    if k.endswith('running_mean'):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
    if k.endswith('bn.bias'):
      sd[k] = 0.1 * torch.randn(sd[k].shape, generator=g)
  coords = _cloud(D, n, D, extent)
  feats = torch.ones(len(coords), cin) if cin == 1 else torch.randn(len(coords), cin, generator=g)
  case = CASES.index((D, cin, cout, k1, normalize, n, extent))
  got = torch.from_numpy(ref_outputs[f'graph_{case}'])          # the reference's forward on these inputs
  want = resunet_forward(sd, coords, feats, k1, normalize)
  assert got.shape == want.shape == (len(coords), cout)
  err = float((got - want).abs().max() / (1 + want.abs().max()))
  assert err <= 1e-6, err
  assert float(want.abs().max()) > 1e-4           # the comparison is not vacuous
