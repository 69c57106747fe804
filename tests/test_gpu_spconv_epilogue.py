"""The line-segment epilogue of the tensor-core sparse convolution (NT >= 128): each consumer warp passes its
fragment through a 16 x 32 shared-memory scratch and adds whole 128-byte row segments with red.global.add.v4.

Pinned to the fp64 criterion of test_gpu_conv_fp64 at every output width where a 32-column block of the scratch is
partly or wholly beyond cout (TF32 cout 80 / 144 / 208, 3xFP16 cout 160 / 224 and the padded 96), on the plain and
the paired list; and a misaligned `out`, which a 16-byte red cannot take, is rejected before any launch.
"""
import pytest
import torch

from test_gpu_conv_fp64 import SIZES, _buckets, _kmap, _data, abi  # noqa: F401
from test_gpu_spconv_runs import N_ROWS, _run_both

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def lists(abi):
  b = _buckets(list(SIZES) * 3, N_ROWS, N_ROWS, seed=11)
  return b, _kmap(abi, b, N_ROWS, N_ROWS, False), _kmap(abi, b, N_ROWS, N_ROWS, True)


@pytest.mark.parametrize('mode,cin,cout', [('tf32', 64, 80), ('tf32', 32, 144), ('tf32', 96, 208),
                                           ('f16', 64, 96), ('f16', 128, 160), ('f16', 192, 224)])
def test_partial_column_blocks(abi, lists, mode, cin, cout):
  b, km, kp = lists
  feat, W = _data(N_ROWS, cin, len(b), cout, seed=cin * 1000 + cout)
  _run_both(abi, mode, feat, W, b, (('plain', km), ('paired', kp)), f'{cin}->{cout}')


def test_misaligned_out_is_rejected(abi):
  f = torch.zeros(256, 64, device='cuda')
  i = torch.zeros(8, dtype=torch.int32, device='cuda')
  o = torch.zeros(4 * 128 + 4, device='cuda')
  P, s = abi.ptr, abi.stream()
  misaligned = P(o) + 4
  bad = [
      ('dgr_spconv_tc_fwd', P(f), 64, P(f), 128, P(i), P(i), P(i), P(i), P(i), 1, 128, 3, misaligned, s),
      ('dgr_spconv_tc_f16_fwd', P(f), 64, P(f), 128, P(i), P(i), P(i), P(i), P(i), 1, 128, P(f), P(f), misaligned, s),
  ]
  for name, *args in bad:
    with pytest.raises(abi.DgrError, match='aligned'):
      abi.call(name, *args)
  torch.cuda.synchronize()
  assert not o.any()
