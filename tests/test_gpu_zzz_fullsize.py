"""BASELINE.json-size checks through size-independent properties (the oracle needs minutes at
these sizes): 3DMatch-shape clouds of ~50k voxels.  Integer work: exact structural invariants;
floating point: adjointness / known answers with the tolerance stated in the test.  Runs last."""
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


@pytest.fixture(scope='module')
def cloud(abi):
  """One full-size scan voxelised on the GPU -> (coords int32 [N, 4] on the device, manager)."""
  from deepglobalregistration_b200.me.coords import CoordinateManager
  xyz = syn.room_scan(0, 250_000)
  d = torch.from_numpy(xyz).cuda()
  raw, _, _, sel, _, n = abi.voxelise(d, 0.05)
  coords = abi.gather_rows_i32(raw, sel, n)
  assert 45_000 <= n <= 55_000, n                   # SURVEY 8(d) config 2
  # voxelisation invariants at full size: ascending first occurrences, one row per voxel
  s = sel[:n].cpu().numpy()
  assert np.all(np.diff(s) > 0)
  c = coords.cpu().numpy()
  assert len(np.unique(c, axis=0)) == n
  assert np.array_equal(c[:, 1:], np.floor(xyz[s] / 0.05).astype(np.int32))
  return coords, CoordinateManager(coords), n


@pytest.mark.parametrize('ks', [3, 7])
def test_kernel_map_structure_full_size(abi, cloud, ks):
  """Bucket kappa and bucket K-1-kappa (offsets o and -o) hold each other's pairs swapped; the centre
  bucket is the identity; every bucket is sorted by output row with each row at most once; the pairs
  satisfy C_in[i] = C_out[j] + offset."""
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  from oracle import sparse_ops as so
  coords, man, n = cloud
  _, km = man.kernel_map(CoordinateMapKey(1), 1, ks)
  K = ks ** 3
  kofs = km.kofs_host
  ii, jj = km.in_idx.cpu().numpy(), km.out_idx.cpu().numpy()
  c = coords.cpu().numpy()[:, 1:].astype(np.int64)
  offs = so.kernel_offsets(ks, 3, 1).astype(np.int64)
  assert km.K == K and int(kofs[K]) == km.n_pairs and km.n_pairs > 10 * n
  mid = K // 2
  assert np.array_equal(ii[kofs[mid]:kofs[mid + 1]], np.arange(n)) and np.array_equal(jj[kofs[mid]:kofs[mid + 1]], np.arange(n))
  for kap in range(K):
    a, b = kofs[kap], kofs[kap + 1]
    i, j = ii[a:b], jj[a:b]
    if b - a > 1:
      assert np.all(np.diff(j) > 0)
    assert np.array_equal(c[i], c[j] + offs[kap])
    ma, mb = kofs[K - 1 - kap], kofs[K - kap]
    mi, mj = ii[ma:mb], jj[ma:mb]
    order = np.argsort(mi, kind='stable')                 # mirrored bucket sorted by ITS input row
    assert np.array_equal(mi[order], j) and np.array_equal(mj[order], i)


def test_conv_adjoint_and_linear_full_size(abi, cloud):
  """<conv(x; W), z> == <x, conv(z; W')> with W'[kappa] = W[K-1-kappa]^T on the same (symmetric) map,
  and conv(2x - 3y) == 2 conv(x) - 3 conv(y): 3xTF32 keeps both to 2e-5 relative at 50k voxels."""
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  coords, man, n = cloud
  _, km = man.kernel_map(CoordinateMapKey(1), 1, 3)
  cin, cout, K = 32, 64, 27
  g = torch.Generator().manual_seed(0)
  W = (torch.randn(K, cin, cout, generator=g) / np.sqrt(cin * 17)).cuda().contiguous()
  Wadj = W.flip(0).transpose(1, 2).contiguous()
  x, y = (torch.randn(n, cin, generator=g).cuda() for _ in range(2))
  z = torch.randn(n, cout, generator=g).cuda()
  Wt, Wt_adj = abi.pack_weight_tf32(W, K, cin, cout), abi.pack_weight_tf32(Wadj, K, cout, cin)

  def conv(v, wt, co):
    out = torch.zeros(n, co, device='cuda')
    abi.spconv_tc_fwd(v.contiguous(), wt, km, out, passes=3)
    return out
  fx, fy = conv(x, Wt, cout), conv(y, Wt, cout)
  lin = conv(2.0 * x - 3.0 * y, Wt, cout)
  scale = float(fx.abs().max())
  assert float((lin - (2.0 * fx - 3.0 * fy)).abs().max()) <= 2e-5 * (1 + 5 * scale)
  back = conv(z, Wt_adj, cin)
  lhs, rhs = float((fx.double() * z.double()).sum()), float((x.double() * back.double()).sum())
  assert abs(lhs - rhs) <= 2e-5 * float((fx.double().abs() * z.double().abs()).sum())
  # and the fp32 FFMA kernel agrees with the tensor-core kernel
  ref = abi.spconv_fwd(x.contiguous(), W, km, torch.zeros(n, cout, device='cuda'))
  assert float((ref - fx).abs().max()) <= 5e-5 * (1 + scale)


def test_knn_tensor_core_equals_fp32_kernel_full_size(abi):
  """51k x 40k x 32 unit-norm features with planted exact duplicates: the wgmma pre-filter path returns
  exactly the fp32 kernel's indices and distances."""
  g = torch.Generator().manual_seed(3)
  n0, n1, c = 51_381, 39_881, 32
  centres = torch.nn.functional.normalize(torch.randn(300, c, generator=g), dim=1)
  F0 = torch.nn.functional.normalize(centres[torch.randint(0, 300, (n0,), generator=g)] + 0.05 * torch.randn(n0, c, generator=g), dim=1)
  F1 = torch.nn.functional.normalize(centres[torch.randint(0, 300, (n1,), generator=g)] + 0.05 * torch.randn(n1, c, generator=g), dim=1)
  F1[777] = F1[55]
  F0[5] = F1[55]
  F0, F1 = F0.cuda().contiguous(), F1.cuda().contiguous()
  i_tc, d_tc = abi.knn_top1(F0, F1, return_distance=True, mode='tc')
  i_ref, d_ref = abi.knn_top1(F0, F1, return_distance=True, mode='simt')
  assert torch.equal(i_tc, i_ref), f'{int((i_tc != i_ref).sum())} rows differ'
  assert torch.equal(d_tc, d_ref)
  assert int(i_tc[5]) == 55                       # lowest index among exact duplicates


def test_register_known_answer_full_size():
  """The rigid-copy known answer (tests/test_gpu_pipeline.py) at BASELINE size: 250k raw points per scan,
  cloud 1 = cloud 0 shifted by a multiple of 8 voxels (voxel 2^-4 m, exact in binary), BatchNorm-calibrated
  random-init checkpoint -> exact correspondences -> the shift recovered to 1e-3 m / 1e-3 rad with ICP
  (2e-3 before it), and reproducibly (integer outputs identical between two runs)."""
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  from deepglobalregistration_b200.util.calibrate import calibrate_batchnorm
  vs = 0.0625
  st = syn.make_checkpoint(4, voxel_size=vs)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))
  xyz0 = syn.room_scan(2, 250_000, scene_seed=1)
  T_gt = np.eye(4)
  T_gt[:3, 3] = vs * np.array([16, -8, 24])
  xyz1 = syn.apply_se3(T_gt, xyz0)
  with torch.no_grad():
    _, c0, f0 = d.preprocess(xyz0)
    calibrate_batchnorm(d.fcgf_model, ME.SparseTensor(f0, coordinates=c0, device='cuda'))
  n0 = len(c0)
  assert n0 > 20_000
  for use_icp in (False, True):
    d.use_icp = use_icp
    T = d.register(xyz0, xyz1)
    assert d.last_branch == 'procrustes' and d.last_info['n0'] == n0
    te, re = syn.rte_rre(T, T_gt)
    # with ICP the rigid copy is matched point for point; before ICP a handful of ambiguous
    # correspondences (near-identical neighbourhoods) may remain in the robust fit: 2e-3 there
    tol = 1e-3 if use_icp else 2e-3
    assert te <= tol and re <= tol, (use_icp, te, re, d.last_info)
  sel_a = d._last_sel.clone()
  d.register(xyz0, xyz1)
  assert torch.equal(sel_a, d._last_sel)
