"""The persistent tensor-core kNN (csrc/knn_tc.cu) against the fp32 brute-force kernel, bit for bit, at the shapes
where its schedule has edges: 128-row tile boundaries, work items that split a row tile or span several, grids
smaller than the SM count, C = 64, every column a candidate, and two streams."""
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def features(n0, n1, c, seed, clustered=True):
  g = torch.Generator().manual_seed(seed)
  if clustered:       # few centres + jitter: several candidates per row
    centres = torch.nn.functional.normalize(torch.randn(40, c, generator=g), dim=1)
    F0 = centres[torch.randint(0, 40, (n0,), generator=g)] + 1e-3 * torch.randn(n0, c, generator=g)
    F1 = centres[torch.randint(0, 40, (n1,), generator=g)] + 1e-3 * torch.randn(n1, c, generator=g)
  else:
    F0 = torch.nn.functional.normalize(torch.randn(n0, c, generator=g), dim=1)
    F1 = torch.nn.functional.normalize(torch.randn(n1, c, generator=g), dim=1)
  return F0.cuda().contiguous(), F1.cuda().contiguous()


def assert_tc_equals_simt(abi, F0, F1):
  i_tc, d_tc = abi.knn_top1(F0, F1, return_distance=True, mode='tc')
  i_ref, d_ref = abi.knn_top1(F0, F1, return_distance=True, mode='simt')
  assert torch.equal(i_tc, i_ref), f'{int((i_tc != i_ref).sum())} rows differ'
  assert torch.equal(d_tc, d_ref)
  return i_tc


# rows at and around one and two 128-row tiles, against tens of thousands of columns and the other way round:
# a CTA's share of the (row tile, column tile) sequence then starts and ends inside a row tile, or spans several
@pytest.mark.parametrize('small', [127, 128, 129, 2 * 128 + 1])
@pytest.mark.parametrize('c', [32, 64])
def test_tile_and_work_item_boundaries_many_columns(abi, small, c):
  assert_tc_equals_simt(abi, *features(small, 40_000 + small, c, seed=small + c))


@pytest.mark.parametrize('small', [127, 128, 129, 2 * 128 + 1])
@pytest.mark.parametrize('c', [32, 64])
def test_tile_and_work_item_boundaries_many_rows(abi, small, c):
  assert_tc_equals_simt(abi, *features(40_000 + small, small, c, seed=3 * small + c))


# fewer (row tile, column tile) pairs than SMs: the grid shrinks to one pair per CTA
@pytest.mark.parametrize('n0,n1,c', [(129, 129, 32), (1, 1, 64), (200, 300, 64), (2, 1000, 32)])
def test_fewer_work_items_than_ctas(abi, n0, n1, c):
  assert_tc_equals_simt(abi, *features(n0, n1, c, seed=n0 + n1, clustered=False))


@pytest.mark.parametrize('c', [32, 64])
def test_identical_features_every_column_a_candidate(abi, c):
  """Every (row, column) pair is a candidate, so the per-warp queues fill and drain many times per tile; the tie
  goes to the lowest column index."""
  row = torch.nn.functional.normalize(torch.randn(1, c, generator=torch.Generator().manual_seed(c)), dim=1)
  F0 = row.expand(1000, c).contiguous().cuda()
  F1 = row.expand(3000, c).contiguous().cuda()
  idx = assert_tc_equals_simt(abi, F0, F1)
  assert int(idx.max()) == 0


def test_two_streams_same_bits(abi):
  F0, F1 = features(30_001, 20_003, 32, seed=7)
  out = []
  for s in (torch.cuda.Stream(), torch.cuda.Stream()):
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
      abi.refresh_stream()
      out.append(abi.knn_top1(F0, F1, return_distance=True, mode='tc'))
    torch.cuda.current_stream().wait_stream(s)
  abi.refresh_stream()
  torch.cuda.synchronize()
  assert torch.equal(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
  i_ref, d_ref = abi.knn_top1(F0, F1, return_distance=True, mode='simt')
  assert torch.equal(out[0][0], i_ref) and torch.equal(out[0][1], d_ref)
