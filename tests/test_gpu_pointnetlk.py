"""dgr_pointnet_forward / dgr_pointnetlk (PointNetLK) against oracle/pointnetlk.py: the fused forward against fp64
under the oracle/precision.py yardstick, the Jacobian, the LK loop stage by stage, the support-function known answer,
the singular exit, argument checks, the baseline, the evaluation entry point and the time per phase."""
import json
import math
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import pointnetlk as ol
from oracle.precision import E32_MIN, KAPPA
from test_oracle_pointnetlk import support_case

pytestmark = pytest.mark.gpu


def _t(a, dtype=torch.float32):
  return torch.as_tensor(np.asarray(a), dtype=dtype).cuda().contiguous()


def _net(sd):
  from deepglobalregistration_b200 import _abi
  from deepglobalregistration_b200.core.pointnetlk import load_pointnet_weights
  packed = _abi.pointnet_pack(_t(load_pointnet_weights(sd), torch.float64))
  return packed, ol.fold(ol.layers_from_state_dict(sd), f32=True)


def _poses(B, seed):
  rng = np.random.default_rng(seed)
  out = [np.eye(4)]
  for _ in range(B - 1):
    out.append(ol.se3_exp(np.concatenate([rng.normal(size=3) * 0.2, rng.normal(size=3) * 0.1])))
  return np.stack(out)


# oracle/precision.py's yardstick with the factor of its whole-network anchor (tests/test_gpu_conv_fp64.py) instead of
# the per-layer KAPPA = 8: each of the four 3xTF32 layers may sit up to ~7x above fp32 (wgmma's accumulator adds do not
# round to nearest) and that compounds.  Measured on one H100 80GB HBM3 (700 W limit), largest e(GPU) / e(fp32) per
# case of test_forward_accuracy: 10.7 (n = 1, B = 1), 15.2 (n = 1, B = 7: one point, so the fp32 error is the
# smallest of the set), 4.4-8.3 for every n >= 127.  The n = 1, B = 7 case sits 5 % under the bar: a change of the
# kernel's accumulation order may put it over, and would then need the accumulation itself made tighter (DESIGN,
# PointNetLK, Accuracy), not a larger factor.
NET_KAPPA = 2 * KAPPA


def feature_bound(folded, inputs):
  """(f64 [B, 1024], bar [B]): the precision yardstick applied to the pooled features of each input cloud."""
  f64, bar = [], []
  for X in inputs:
    a = ol.phi(folded, X)
    b = ol.phi(folded, X, np.float32).astype(np.float64)
    f64.append(a)
    bar.append(NET_KAPPA * max(np.abs(b - a).max(), E32_MIN * np.abs(a).max()))
  return np.stack(f64), np.array(bar)


@pytest.mark.parametrize('n', [1, 127, 128, 129, 1000, 51381])
@pytest.mark.parametrize('B', [1, 7])
def test_forward_accuracy(n, B):
  from deepglobalregistration_b200 import _abi
  packed, folded = _net(syn.pointnetlk_state_dict(n % 97))
  P = (syn.room_scan(n % 13, n_raw=n) - np.array([1.8, 1.5, 1.2])).astype(np.float32)
  c = np.array([0.05, -0.02, 0.01])
  G = _poses(B, n)
  f = _abi.pointnet_forward(_t(P), _t(G, torch.float64), packed, centre=_t(c, torch.float64))
  f2 = _abi.pointnet_forward(_t(P), _t(G, torch.float64), packed, centre=_t(c, torch.float64))
  f, f2 = f.cpu().numpy(), f2.cpu().numpy()
  assert np.array_equal(f.view(np.uint32), f2.view(np.uint32))
  f64, bar = feature_bound(folded, [ol.transform32(P, g, c) for g in G])
  err = np.abs(f.astype(np.float64) - f64).max(axis=1)
  print(f'\n[pointnetlk] forward n={n} B={B}: e(GPU) / e(fp32) = {(err / bar * NET_KAPPA).max():.2f} '
        f'(bar {NET_KAPPA:g}); max f {f64.max():.3g}')
  assert (f >= 0).all() and (err <= bar).all(), (err, bar)


def test_jacobian():
  from deepglobalregistration_b200 import _abi
  sd = syn.pointnetlk_state_dict(5)
  packed, folded = _net(sd)
  P, Q, _ = support_case(5.0, 5.0, 2000)
  delta = 1e-2
  _, J = _abi.pointnetlk(_t(P), _t(Q), packed, delta=delta, max_iter=1, return_jacobian=True)
  J = J.cpu().numpy()
  mt = ol.stats_mean(Q)
  poses = np.stack(ol.jacobian_poses(delta))
  fj = _abi.pointnet_forward(_t(Q), _t(poses, torch.float64), packed, centre=_t(mt, torch.float64)).cpu().numpy()
  J_own = ol.jacobian(fj, delta)
  f64, bar = feature_bound(folded, [ol.transform32(Q, g, mt) for g in poses])
  J64 = ol.jacobian(f64, delta)
  own = np.abs(J - J_own).max()
  exact = (J == J_own).mean()
  print(f'\n[pointnetlk] J: {100 * exact:.2f} % of entries equal to J from the GPU features, max diff {own:.3g}; '
        f'max |J - J64| {np.abs(J - J64).max():.3g} vs bar {2 * bar.max() / delta:.3g}')
  # the GPU's exp(-delta e_i) comes from CUDA's sin / cos: a last-bit difference may move a rounded input point
  assert own <= 2 * bar.max() / delta and exact > 0.5
  assert np.abs(J - J64).max() <= 2 * bar.max() / delta


def _lk_parity(sd, P, Q, label, max_iter=10, xtol=1e-7):
  """Stage-isolated parity.  The oracle takes every step from the GPU's own numbers: J from jac_out, and f0 and the
  features at each logged g_k from dgr_pointnet_forward with the same pose bits and the same centre (the same network
  inputs, so the same feature bits as inside the call).  It must land on the GPU's g_{k+1} to 1e-9: what is left
  between the two is the fp64 solve (the library's fixed-order sums and 6x6 Cholesky against numpy's).  |r| and |dx|
  must agree to 1e-10 / 1e-6 relative, and the stop decision (|dx| < xtol) at every step, so the iteration counts
  agree, except where |dx| lies within 1e-3 relative of xtol.  The full oracle run on its own fp64 features is a
  printed secondary comparison: the GPU features' fp32 error moves |dx| near convergence, so that run may stop a step
  apart."""
  from deepglobalregistration_b200 import _abi
  packed, folded = _net(sd)
  delta = 1e-2
  res, J, log = _abi.pointnetlk(_t(P), _t(Q), packed, delta=delta, max_iter=max_iter, xtol=xtol,
                                return_jacobian=True, return_log=True)
  res2, J2, log2 = _abi.pointnetlk(_t(P), _t(Q), packed, delta=delta, max_iter=max_iter, xtol=xtol,
                                   return_jacobian=True, return_log=True)
  res, J, log = res.cpu().numpy(), J.cpu().numpy(), log.cpu().numpy()
  assert np.array_equal(res, res2.cpu().numpy()) and np.array_equal(J, J2.cpu().numpy())
  assert np.array_equal(log, log2.cpu().numpy(), equal_nan=True)
  info = dict(zip(_abi.POINTNETLK_RESULT, res[16:23]))
  assert info['status'] == 0 and info['host_reads'] == 0
  it = int(info['iterations'])
  assert 1 <= it <= max_iter and np.isnan(log[it:]).all() and not np.isnan(log[:it]).any()
  ms, mt = ol.stats_mean(P), ol.stats_mean(Q)
  f0 = _abi.pointnet_forward(_t(Q), _t(np.eye(4)[None], torch.float64), packed,
                             centre=_t(mt, torch.float64)).cpu().numpy()[0]
  H = J.T @ J
  gs = np.tile(np.eye(4), (it, 1, 1))
  gs[:, :3] = log[:it, :12].reshape(it, 3, 4)
  F = _abi.pointnet_forward(_t(P), _t(gs, torch.float64), packed, centre=_t(ms, torch.float64)).cpu().numpy()
  T_last = res[:16].reshape(4, 4)
  g_final = np.eye(4)                       # the final g, back in the centred frames
  g_final[:3, :3] = T_last[:3, :3]
  g_final[:3, 3] = T_last[:3, 3] + T_last[:3, :3] @ ms - mt
  worst = dict(g=0.0, r=0.0, dx=0.0)
  for k in range(it):
    dx, ndx, nr = ol.step(J, H, F[k], f0)
    worst['r'] = max(worst['r'], abs(nr - log[k, 13]) / nr)
    worst['dx'] = max(worst['dx'], abs(ndx - log[k, 12]) / ndx)
    assert abs(nr - log[k, 13]) <= 1e-10 * nr and abs(ndx - log[k, 12]) <= 1e-6 * ndx, (label, k, nr, ndx, log[k])
    near = abs(ndx - xtol) <= 1e-3 * xtol
    assert near or (ndx < xtol) == (log[k, 12] < xtol), (label, k, ndx, log[k, 12])
    assert k == it - 1 or log[k, 12] >= xtol                 # the library runs on until its |dx| < xtol
    if log[k, 12] < xtol:                  # the library stopped here: its pose is g_k
      diff = np.abs(g_final - gs[k]).max()
    else:
      diff = np.abs(ol.se3_exp(dx) @ gs[k] - (gs[k + 1] if k + 1 < it else g_final)).max()
    worst['g'] = max(worst['g'], diff)
    assert diff <= 1e-9, (label, k, diff)
  T_o, info_o, _, _ = ol.pointnetlk(P, Q, folded, delta=delta, max_iter=max_iter, xtol=xtol)
  print(f'\n[pointnetlk] {label}: {it} iterations, largest differences from the oracle stepped on the GPU\'s '
        f'features: g {worst["g"]:.3g}, |r| {worst["r"]:.3g} rel, |dx| {worst["dx"]:.3g} rel; the oracle on its own '
        f'fp64 features: {info_o["iterations"]} iterations, |T - T_oracle| {np.abs(T_last - T_o).max():.3g}')
  return T_last, T_o, info


def test_lk_stage_parity_random_network():
  sd = syn.pointnetlk_state_dict(7)
  P, Q, _ = support_case(4.0, 4.0, 2000)
  _lk_parity(sd, P, Q, 'random network')


def test_support_function_known_answer_on_the_gpu():
  sd = syn.pointnetlk_support_state_dict()
  P, Q, T_gt = support_case()
  T, T_o, info = _lk_parity(sd, P, Q, 'support function')
  te, re = syn.rte_rre(T, T_o)
  print(f'[pointnetlk] support function: {te:.3g} m / {re:.3g} rad from the oracle, {syn.rte_rre(T, T_gt)} from truth')
  assert te <= 1e-4 and re <= 1e-4 and info['iterations'] < 10


def test_singular_network_returns_the_centroid_alignment():
  from deepglobalregistration_b200 import _abi
  sd = syn.pointnetlk_state_dict(0)
  sd['h2.6.weight'].zero_()
  packed, _ = _net(sd)
  P = syn.room_scan(0, n_raw=2000).astype(np.float32)
  Q = P + np.float32([0.3, -0.2, 0.1])
  res, J = _abi.pointnetlk(_t(P), _t(Q), packed, return_jacobian=True)
  res = res.cpu().numpy()
  info = dict(zip(_abi.POINTNETLK_RESULT, res[16:23]))
  assert info['status'] == 1 and info['iterations'] == 0 and not J.cpu().numpy().any()
  expect = np.eye(4)
  expect[:3, 3] = ol.stats_mean(Q) - ol.stats_mean(P)
  assert np.array_equal(res[:16].reshape(4, 4), expect)


def test_bad_arguments_raise():
  from deepglobalregistration_b200 import _abi
  packed, _ = _net(syn.pointnetlk_state_dict(0))
  P = _t(syn.room_scan(0, n_raw=200))
  for kw in (dict(delta=0.0), dict(delta=float('inf')), dict(max_iter=0), dict(max_iter=1001), dict(xtol=-1.0)):
    with pytest.raises(_abi.DgrError):
      _abi.pointnetlk(P, P, packed, **kw)
  with pytest.raises(_abi.DgrError):
    _abi.pointnetlk(P[:0], P, packed)
  with pytest.raises(_abi.DgrError):
    _abi.pointnet_forward(P[:0], _t(np.eye(4)[None], torch.float64), packed)
  with pytest.raises(_abi.DgrError):
    _abi.pointnet_pack(torch.zeros(10, dtype=torch.float64, device='cuda'))
  eye = _t(np.eye(4)[None], torch.float64)
  for bad in (packed[:-16], packed.float(), torch.zeros(packed.numel() + 16, dtype=torch.uint8, device='cuda')[8:-8]):
    with pytest.raises(_abi.DgrError):
      _abi.pointnet_forward(P, eye, bad)
    with pytest.raises(_abi.DgrError):
      _abi.pointnetlk(P, P, bad)
  for poses in (eye[0], _t(np.zeros((1, 3, 3)), torch.float64)):
    with pytest.raises(_abi.DgrError):
      _abi.pointnet_forward(P, poses, packed)


def test_nan_point_makes_nan_features():
  """A NaN input point propagates through the ReLUs and the max, as in the oracle (np.maximum / np.max keep NaN)."""
  from deepglobalregistration_b200 import _abi
  packed, folded = _net(syn.pointnetlk_state_dict(2))
  P = (syn.room_scan(2, n_raw=300) - 1.5).astype(np.float32)
  P[137, 1] = np.nan
  G = _poses(2, 3)
  f = _abi.pointnet_forward(_t(P), _t(G, torch.float64), packed).cpu().numpy()
  assert np.isnan(ol.phi(folded, ol.transform32(P, G[0]))).all() and np.isnan(f).all()
  P[137, 1] = 0.0
  assert np.isfinite(_abi.pointnet_forward(_t(P), _t(G, torch.float64), packed).cpu().numpy()).all()


def _dgr(vs=0.0625):
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  st = syn.make_checkpoint(4, voxel_size=vs)
  return DeepGlobalRegistration(types.SimpleNamespace(weights=st, clip_weight_thresh=0.05, verbose=False))


def test_baseline_on_a_room_pair(tmp_path):
  from deepglobalregistration_b200.core.pointnetlk import PointNetLKBaseline
  torch.save(syn.pointnetlk_support_state_dict(), tmp_path / 'pnlk.pth')
  xyz0, xyz1, T_gt = syn.room_pair(3, n_raw=60_000)
  b = PointNetLKBaseline(_dgr(), str(tmp_path / 'pnlk.pth'))
  T = b.register(xyz0, xyz1)
  te, re = syn.rte_rre(T, T_gt)
  print(f'\n[pointnetlk] baseline (support-function network): rte {te:.4f} m, rre {math.degrees(re):.3f} deg, '
        f'{b.last_info}')
  assert b.last_branch == 'pointnetlk' and b.last_info['status'] == 0 and 1 <= b.last_info['iterations'] <= 10
  # measured on one H100 80GB HBM3: 0.0213 m / 0.398 deg after 10 iterations (two independent samplings of the room, so
  # the support functions differ by the sampling); the bar sits about 2.5x above
  assert te < 0.05 and math.degrees(re) < 1.0, (te, math.degrees(re), b.last_info)


def test_evaluate_pointnetlk_on_a_pair_list(tmp_path, capsys):
  from deepglobalregistration_b200 import evaluate as ev
  from deepglobalregistration_b200 import io as dio
  torch.save(syn.make_checkpoint(0), tmp_path / 'ckpt.pth')
  torch.save(syn.pointnetlk_state_dict(0), tmp_path / 'pnlk.pth')
  lines = []
  for k in range(2):
    xyz0, xyz1, T_gt = syn.room_pair(k, n_raw=30_000)
    np.savez(tmp_path / f'a{k}.npz', pcd=xyz0)
    dio.write_ply(tmp_path / f'b{k}.ply', xyz1, dtype='double')
    lines.append(f'a{k}.npz b{k}.ply {" ".join(repr(float(x)) for x in T_gt.reshape(-1))} room')
  (tmp_path / 'pairs.txt').write_text('\n'.join(lines) + '\n')
  ev.main(['--pair_list', str(tmp_path / 'pairs.txt'), '--weights', str(tmp_path / 'ckpt.pth'), '--out_dir',
           str(tmp_path), '--method', 'pointnetlk', '--pointnetlk_weights', str(tmp_path / 'pnlk.pth'),
           '--pointnetlk_max_iter', '5'])
  summary = json.loads(capsys.readouterr().out.strip().splitlines()[-1])
  assert summary['pairs'] == 2 and summary['with_ground_truth'] == 2
  saved = np.load(tmp_path / 'pointnetlk-b200-stats.npz', allow_pickle=True)
  assert list(saved['names']) == ['PointNetLK'] and saved['stats'].shape == (1, 2, 5)


def test_dgr_size_pair_timing():
  """room_pair(0) at the bench's voxel size (about 51k / 40k voxels): one forward, the 7-pose Jacobian forward,
  one LK iteration and the whole call (CUDA events); correctness only, no speed bar."""
  from deepglobalregistration_b200 import _abi
  from deepglobalregistration_b200.core.pointnetlk import PointNetLKBaseline
  xyz0, xyz1, _ = syn.room_pair(0)
  b = PointNetLKBaseline(_dgr(0.05), syn.pointnetlk_state_dict(0))
  b.register(xyz0, xyz1)
  p0, _, _ = b.dgr.preprocess(xyz0, 0, _batch=0)
  p1, _, _ = b.dgr.preprocess(xyz1, 1, _batch=1)
  src, tgt = p0.float().contiguous(), p1.float().contiguous()
  I = _t(np.eye(4)[None], torch.float64)
  J7 = _t(np.stack(ol.jacobian_poses(1e-2)), torch.float64)

  def timed(fn, reps=5):
    fn()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(reps):
      fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / reps

  t1 = timed(lambda: _abi.pointnet_forward(src, I, b.packed))
  t7 = timed(lambda: _abi.pointnet_forward(tgt, J7, b.packed))
  t_call = timed(lambda: _abi.pointnetlk(src, tgt, b.packed, max_iter=10, xtol=0.0))
  t_one = timed(lambda: _abi.pointnetlk(src, tgt, b.packed, max_iter=1, xtol=0.0))
  res = _abi.pointnetlk(src, tgt, b.packed, max_iter=10, xtol=0.0).cpu().numpy()
  print(f'\n[pointnetlk] n_src {len(src)}, n_tgt {len(tgt)}: forward {t1:.3f} ms, 7-pose forward {t7:.3f} ms, '
        f'one LK iteration {(t_call - t_one) / 9:.3f} ms, whole call (10 iterations) {t_call:.3f} ms')
  assert len(src) > 30000 and res[16] == 10
