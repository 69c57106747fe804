"""oracle/pointnetlk.py (CPU): the network against a torch.nn stack, the SE(3) exponential against expm, the LK loop's
exits, the support-function known answer, and the checkpoint loader's rejections."""
import math

import numpy as np
import pytest
import scipy.linalg
import torch

from deepglobalregistration_b200 import synthetic as syn
from deepglobalregistration_b200.core.pointnetlk import load_pointnet_weights
from oracle import pointnetlk as ol


def torch_stack(sd):
  """The published PointNet_features layout built from torch.nn modules, eval mode, fp64."""
  mods = []
  for (conv, bn), (cin, cout) in zip(ol.MODULES, ol.WIDTHS):
    c, b = torch.nn.Conv1d(cin, cout, 1), torch.nn.BatchNorm1d(cout, eps=1e-5)
    c.weight.data, c.bias.data = sd[conv + '.weight'].clone(), sd[conv + '.bias'].clone()
    for k in ('weight', 'bias', 'running_mean', 'running_var'):
      getattr(b, k).data = sd[f'{bn}.{k}'].clone()
    mods += [c, b, torch.nn.ReLU()]
  return torch.nn.Sequential(*mods).double().eval()


def support_case(deg=10.0, cm=10.0, n_raw=3000, seed=0):
  """A room scan and its exact rigid copy, turned by `deg` about its centroid and moved by `cm`."""
  P = syn.room_scan(seed, n_raw=n_raw).astype(np.float32)
  c = P.astype(np.float64).mean(0)
  rng = np.random.default_rng(int(deg))
  ax = rng.normal(size=3)
  ax /= np.linalg.norm(ax)
  T = ol.se3_exp(np.concatenate([ax * math.radians(deg), np.zeros(3)]))
  d = rng.normal(size=3)
  T[:3, 3] = d / np.linalg.norm(d) * cm / 100 + c - T[:3, :3] @ c
  return P, syn.apply_se3(T, P.astype(np.float64)).astype(np.float32), T


def test_phi_matches_a_torch_stack():
  sd = syn.pointnetlk_state_dict(3)
  X = syn.room_scan(1, n_raw=500) - 1.5
  ref = torch_stack(sd)(torch.from_numpy(X.T[None].copy())).max(dim=2).values[0].detach().numpy()
  layers = ol.layers_from_state_dict(sd)
  got = ol.phi(ol.fold(layers), X)
  assert np.abs(got - ref).max() <= 1e-12 * np.abs(ref).max()
  # the folded network equals the unfolded one layer by layer
  h = X
  for W, b, g, beta, mean, var in layers:
    h = np.maximum((h @ W.T + b - mean) / np.sqrt(var + ol.EPS) * g + beta, 0.0)
  assert np.abs(got - h.max(0)).max() <= 1e-12 * np.abs(ref).max()
  assert (got >= 0).all() and got.max() > 0


@pytest.mark.parametrize('theta', [1e-9, 5e-3, 1.0, math.pi - 1e-6])
def test_exp_matches_expm(theta):
  rng = np.random.default_rng(int(theta * 1e6) % 1000)
  w = rng.normal(size=3)
  w *= theta / np.linalg.norm(w)
  v = rng.normal(size=3)
  M = np.zeros((4, 4))
  M[:3, :3] = [[0, -w[2], w[1]], [w[2], 0, -w[0]], [-w[1], w[0], 0]]
  M[:3, 3] = v
  assert np.abs(ol.se3_exp(np.concatenate([w, v])) - scipy.linalg.expm(M)).max() <= 1e-12


def test_identical_clouds_stop_at_once():
  folded = ol.fold(ol.layers_from_state_dict(syn.pointnetlk_state_dict(0)), f32=True)
  P = syn.room_scan(0, n_raw=2000).astype(np.float32)
  T, info, log, _ = ol.pointnetlk(P, P, folded)
  assert info['status'] == 0 and info['iterations'] == 1 and info['last_dx'] == 0.0 and info['last_r'] == 0.0
  assert np.array_equal(T, np.eye(4)) and len(log) == 1


def test_zero_last_layer_is_singular():
  sd = syn.pointnetlk_state_dict(0)
  sd['h2.6.weight'].zero_()
  folded = ol.fold(ol.layers_from_state_dict(sd), f32=True)
  P = syn.room_scan(0, n_raw=2000).astype(np.float32)
  Q = P + np.float32([0.3, -0.2, 0.1])
  T, info, log, J = ol.pointnetlk(P, Q, folded)
  assert info['status'] == 1 and info['iterations'] == 0 and len(log) == 0 and not J.any()
  expect = np.eye(4)
  expect[:3, 3] = ol.stats_mean(Q) - ol.stats_mean(P)
  assert np.array_equal(T, expect)


def test_support_function_known_answer():
  """Measured with this oracle on this case (n = 3000, 10 deg, 10 cm, defaults): 6 iterations, 6.5e-8 m and
  8.5e-7 deg from the true pose; the same case at 30 deg still ends within 1.1e-7 m / 2.1e-6 deg in 7 iterations
  (max_iter 20).  The bars sit 10x above the 10 deg measurement."""
  folded = ol.fold(ol.layers_from_state_dict(syn.pointnetlk_support_state_dict()), f32=True)
  P, Q, T_gt = support_case()
  T, info, _, _ = ol.pointnetlk(P, Q, folded)
  te, re = syn.rte_rre(T, T_gt)
  assert info['status'] == 0 and info['iterations'] < 10 and info['last_dx'] < 1e-7
  assert te < 1e-6 and math.degrees(re) < 1e-5, (te, math.degrees(re), info)
  # the features are the support function, up to the constant offset and fp32 weights
  A = syn.fibonacci_sphere(1024)
  Pc = P.astype(np.float64) - P.astype(np.float64).mean(0)
  f = ol.phi(folded, ol.transform32(P, np.eye(4), P.astype(np.float64).mean(0)))
  assert np.abs(f - ((Pc @ A.T).max(0) + 10.0)).max() < 1e-4


def test_loader_accepts_prefixes_and_rejects_bad_state_dicts(tmp_path):
  sd = syn.pointnetlk_state_dict(1)
  ref = load_pointnet_weights(sd)
  assert ref.shape == (154368,) and ref.dtype == np.float64
  torch.save({f'module.ptnet.{k}': v for k, v in sd.items()} | {'dt': torch.ones(1, 6)}, tmp_path / 'w.pth')
  assert np.array_equal(load_pointnet_weights(str(tmp_path / 'w.pth')), ref)
  bad = dict(sd)
  del bad['h1.1.running_var']
  with pytest.raises(ValueError, match=r'missing \[.h1\.1\.running_var.\]'):
    load_pointnet_weights(bad)
  bad = dict(sd, **{'h3.0.weight': torch.zeros(1)})
  with pytest.raises(ValueError, match=r'unexpected \[.h3\.0\.weight.\]'):
    load_pointnet_weights(bad)
  bad = dict(sd, **{'h2.6.weight': torch.zeros(512, 128, 1)})
  with pytest.raises(ValueError, match=r'h2\.6\.weight \(512, 128, 1\)'):
    load_pointnet_weights(bad)


def test_evaluate_refuses_pointnetlk_without_weights(capsys):
  from deepglobalregistration_b200 import evaluate as ev
  with pytest.raises(SystemExit):
    ev.main(['--pair_list', 'pairs.txt', '--weights', 'ckpt.pth', '--method', 'pointnetlk'])
  assert '--pointnetlk_weights' in capsys.readouterr().err
