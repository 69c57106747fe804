"""Round-2 native layer: coordinate planning with device-side counts (csrc/coordplan.cu) and the native
executor (csrc/exec.cu) against the operator path and the CPU oracle.

Integer work is bit-exact (coarse maps, kernel-map pair lists, voxel selection); floating point within the
stated tolerances (atomic scatter-add order differs between runs: 2e-5 relative)."""
import ctypes as C
import types

import numpy as np
import pytest
import torch

from deepglobalregistration_b200 import synthetic as syn
from oracle import sparse_ops as so

pytestmark = pytest.mark.gpu


@pytest.fixture(scope='module')
def abi():
  from deepglobalregistration_b200 import _abi
  _abi.require_device('cuda')
  return _abi


def _cloud(D, n, ext, seed, batch2=False):
  g = np.random.default_rng(seed)
  c = np.unique(g.integers(-ext, ext, size=(n, D)), axis=0)
  c = c[g.permutation(len(c))]
  b = np.zeros((len(c), 1), np.int64) if not batch2 else g.integers(0, 2, size=(len(c), 1))
  return np.concatenate([b, c], 1).astype(np.int32)


def _spec_and_table(abi, coords_t):
  from deepglobalregistration_b200.me.coords import CoordinateManager
  man = CoordinateManager(coords_t, assume_unique=True)
  return man, man.spec, man._maps[1].table


def _padded(coords, extra, seed=1):
  """coords followed by `extra` garbage rows: the device-side count must hide them."""
  g = np.random.default_rng(seed)
  junk = g.integers(-3, 3, size=(extra, coords.shape[1])).astype(np.int32)
  junk[:, 0] = 0
  return torch.from_numpy(np.concatenate([coords, junk], 0)).cuda().contiguous()


@pytest.mark.parametrize('D,n,ext', [(3, 6000, 14), (6, 5000, 3), (3, 40, 3)])
def test_coarse_maps_device_count_bit_exact(abi, D, n, ext):
  coords = _cloud(D, n, ext, seed=D + n, batch2=True)
  nreal = len(coords)
  ct = torch.from_numpy(coords).cuda().contiguous()
  man, spec, _ = _spec_and_table(abi, ct)
  n_max = nreal + 777
  pad = _padded(coords, 777)
  n_dev = torch.tensor([nreal], dtype=torch.int32, device='cuda')
  cap = max(1024, abi.next_pow2(2 * n_max))
  L, ncols = 3, D + 1
  keys = torch.empty(L, cap, dtype=torch.int64, device='cuda')
  vals = torch.empty(L, cap, dtype=torch.int32, device='cuda')
  out = torch.full((L, n_max, ncols), -77, dtype=torch.int32, device='cuda')
  n_out = torch.zeros(L, dtype=torch.int32, device='cuda')
  slot = torch.empty(L * n_max, dtype=torch.int32, device='cuda')
  scan = torch.empty(L * abi.lib().dgr_scan_ws_elems(n_max), dtype=torch.int32, device='cuda')
  strides = (C.c_int32 * 3)(2, 4, 8)
  abi.call('dgr_coarse_maps', abi.ptr(pad), n_max, abi.ptr(n_dev), ncols, abi.ptr(spec), L, strides, abi.ptr(keys),
           abi.ptr(vals), cap, abi.ptr(out), abi.ptr(n_out), abi.ptr(slot), abi.ptr(scan), abi.stream())
  torch.cuda.synchronize()
  counts = n_out.cpu().tolist()
  fine = coords
  for l, s in enumerate((2, 4, 8)):
    want, _ = so.stride_coords(fine, s)            # cascaded, as ME builds them; ours derives from stride 1
    fine = want
    got = out[l, :counts[l]].cpu().numpy()
    assert counts[l] == len(want)
    assert np.array_equal(got, want), (D, s)
    # the table maps every coarse key to its row
    rows = abi.hash_find(torch.from_numpy(want).cuda().contiguous(), spec,
                         types.SimpleNamespace(keys=keys[l], vals=vals[l], cap=cap))
    assert torch.equal(rows.cpu(), torch.arange(len(want), dtype=torch.int32))


def _new_kmap(abi, out_coords, n_out_max, n_out_dev, spec, table, offsets, bloom):
  K, ncols = offsets.shape[0], out_coords.shape[1]
  W = abi.lib().dgr_kmap_mask_words(n_out_max)
  bits = torch.full((K * W,), -1, dtype=torch.int32, device='cuda')          # poisoned: every word must be written
  cnt = torch.empty(abi.lib().dgr_kmap_cnt_elems(K, n_out_max), dtype=torch.int32, device='cuda')
  kofs = torch.empty(K + 2, dtype=torch.int32, device='cuda')
  meta = torch.empty(5, dtype=torch.int32, device='cuda')
  words, n_words = None, 0
  if bloom:
    n_words = 4096
    words = torch.empty(n_words, dtype=torch.int32, device='cuda')
    abi.call('dgr_bloom2_build', abi.ptr(table.keys), table.cap, abi.ptr(words), n_words, abi.stream())
  abi.call('dgr_kmap_probe', abi.ptr(out_coords), n_out_max, abi.ptr(n_out_dev), ncols, abi.ptr(spec), abi.ptr(table.keys),
           abi.ptr(table.vals), table.cap, abi.ptr(words), n_words, abi.ptr(offsets), K, abi.ptr(bits), abi.ptr(cnt),
           abi.ptr(kofs), abi.ptr(meta), abi.stream())
  m = meta.cpu().tolist()
  P = m[0]
  in_idx = torch.empty(max(P, 1), dtype=torch.int32, device='cuda')
  out_idx = torch.empty(max(P, 1), dtype=torch.int32, device='cuda')
  abi.call('dgr_kmap_fill', abi.ptr(bits), abi.ptr(cnt), K, n_out_max, abi.ptr(out_coords), ncols, abi.ptr(spec),
           abi.ptr(table.keys), abi.ptr(table.vals), table.cap, abi.ptr(offsets), abi.ptr(in_idx), abi.ptr(out_idx),
           abi.stream())
  torch.cuda.synchronize()
  return kofs.cpu().numpy(), in_idx[:P].cpu().numpy(), out_idx[:P].cpu().numpy(), m


def _bucket_offsets(buckets):
  return np.concatenate([[0], np.cumsum([len(b[0]) for b in buckets])])


def _dense_table(buckets, n_out):
  """nbr[kappa, j] = i for every pair of bucket kappa, otherwise -1."""
  nbr = np.full((len(buckets), n_out), -1, np.int32)
  for kap, (i, j) in enumerate(buckets):
    nbr[kap, j] = i
  return nbr


@pytest.mark.parametrize('D,ks,n,ext,bloom', [(3, 3, 9000, 16, False), (3, 5, 3000, 9, False), (6, 3, 6000, 3, True),
                                              (6, 3, 6000, 3, False), (3, 3, 30, 2, False)])
def test_kernel_map_bits_equal_oracle_buckets(abi, D, ks, n, ext, bloom):
  from deepglobalregistration_b200.me.coords import kernel_offsets
  coords = _cloud(D, n, ext, seed=ks + n)
  ct = torch.from_numpy(coords).cuda().contiguous()
  man, spec, table = _spec_and_table(abi, ct)
  offs = kernel_offsets(ks, D, 1, torch.device('cuda'))
  buckets = so.kernel_map(coords, coords, so.kernel_offsets(ks, D, 1))
  want_kofs = _bucket_offsets(buckets)
  counts = np.diff(want_kofs)
  tiles = (counts + 127) // 128
  want_i = np.concatenate([b[0] for b in buckets])
  want_j = np.concatenate([b[1] for b in buckets])
  nreal = len(coords)
  for extra in (0, 1500):
    n_max = nreal + extra
    oc = _padded(coords, extra) if extra else ct
    n_dev = torch.tensor([nreal], dtype=torch.int32, device='cuda')
    kofs, ii, jj, meta = _new_kmap(abi, oc, n_max, n_dev, spec, table, offs, bloom)
    K = ks ** D
    assert np.array_equal(kofs[:K + 1], want_kofs)
    assert meta[0] == want_kofs[-1] and meta[1] == tiles.sum() and meta[2] == ((tiles + 1) // 2 * 2).sum()
    assert meta[3] == int((counts > 0).sum()) and meta[4] == 0
    assert np.array_equal(ii, want_i)
    assert np.array_equal(jj, want_j)


def test_strided_kernel_map_and_dense_table(abi):
  from deepglobalregistration_b200.me.coords import CoordinateMapKey, kernel_offsets
  coords = _cloud(3, 8000, 15, seed=5)
  ct = torch.from_numpy(coords).cuda().contiguous()
  man, spec, table = _spec_and_table(abi, ct)
  _, km = man.kernel_map(CoordinateMapKey(1), 2, 3)                 # stride-2 convolution map 1 -> 2
  coarse = man.coordinates(CoordinateMapKey(2))
  offs = kernel_offsets(3, 3, 1, torch.device('cuda'))
  n2 = coarse.shape[0]
  kofs, ii, jj, meta = _new_kmap(abi, coarse, n2, None, spec, table, offs, False)
  down = so.kernel_map(coords, coarse.cpu().numpy(), so.kernel_offsets(3, 3, 1))
  assert np.array_equal(kofs[:28], _bucket_offsets(down)) and np.array_equal(kofs[:28], km.kofs_host)
  assert np.array_equal(ii, np.concatenate([b[0] for b in down]))
  assert np.array_equal(jj, np.concatenate([b[1] for b in down]))
  assert np.array_equal(ii, km.in_idx[:km.n_pairs].cpu().numpy())
  assert np.array_equal(jj, km.out_idx[:km.n_pairs].cpu().numpy())
  # dense table with a row stride and a device count
  offs7 = kernel_offsets(7, 3, 1, torch.device('cuda'))
  n = len(coords)
  b7 = so.kernel_map(coords, coords, so.kernel_offsets(7, 3, 1))
  want = torch.from_numpy(_dense_table(b7, n)).cuda()
  stride = n + 100
  nbr = torch.full((343, stride), -5, dtype=torch.int32, device='cuda')
  n_dev = torch.tensor([n], dtype=torch.int32, device='cuda')
  padded = _padded(coords, 100)
  abi.call('dgr_kmap_dense', abi.ptr(padded), n + 100, abi.ptr(n_dev), 4, abi.ptr(spec), abi.ptr(table.keys),
           abi.ptr(table.vals), table.cap, None, 0, abi.ptr(offs7), 343, abi.ptr(nbr), stride, None, abi.stream())
  assert torch.equal(nbr[:, :n], want) and bool((nbr[:, n:] == -5).all())
  # with the shared-memory miss filter
  words = torch.empty(2048, dtype=torch.int32, device='cuda')
  abi.call('dgr_bloom2_build', abi.ptr(table.keys), table.cap, abi.ptr(words), 2048, abi.stream())
  nbr2 = torch.full((343, stride), -5, dtype=torch.int32, device='cuda')
  hits = torch.full((1,), 77, dtype=torch.int32, device='cuda')
  abi.call('dgr_kmap_dense', abi.ptr(padded), n + 100, abi.ptr(n_dev), 4, abi.ptr(spec), abi.ptr(table.keys),
           abi.ptr(table.vals), table.cap, abi.ptr(words), 2048, abi.ptr(offs7), 343, abi.ptr(nbr2), stride, abi.ptr(hits),
           abi.stream())
  assert torch.equal(nbr2[:, :n], want) and bool((nbr2[:, n:] == -5).all())
  assert int(hits) == sum(len(b[0]) for b in b7)


@pytest.fixture(scope='module')
def dgr():
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  state = syn.make_checkpoint(0)
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
  d.use_icp = False
  return d, state


@pytest.mark.parametrize('which,ks', [('fcgf', 7), ('fcgf', 5), ('fcgf', 3), ('inlier', 3), ('inlier_coords', 3)])
def test_native_net_forward_matches_operator_path(abi, dgr, which, ks):
  from deepglobalregistration_b200 import native
  from deepglobalregistration_b200 import me as ME
  from deepglobalregistration_b200.model import load_model
  d, state = dgr
  if which == 'fcgf':
    sd = syn.resunet_state_dict(11, 1, 32, ks, 3)
    model = load_model('ResUNetBN2C')(1, 32, bn_momentum=0.05, conv1_kernel_size=ks, normalize_feature=True, D=3)
    model.load_state_dict(sd)
    model = model.cuda().eval()
    coords = _cloud(3, 7000, 12, seed=ks, batch2=True)
  elif which == 'inlier':
    model = d.inlier_model
    coords = _cloud(6, 5000, 3, seed=9)
  else:                     # the 'coords' inlier feature type: six input channels, cos of both points
    model = load_model('ResUNetBN2C')(6, 1, bn_momentum=0.05, conv1_kernel_size=ks, normalize_feature=False, D=6)
    model.load_state_dict(syn.resunet_state_dict(12, 6, 1, ks, 6))
    model = model.cuda().eval()
    coords = _cloud(6, 5000, 3, seed=10)
  ct = torch.from_numpy(coords).cuda().contiguous()
  g = torch.Generator().manual_seed(ks)
  feats = torch.ones(len(coords), 1) if model.conv1.in_channels == 1 else torch.cos(3 * torch.randn(len(coords), 6, generator=g))
  feats = feats.cuda().contiguous()
  with torch.no_grad():
    want = model(ME.SparseTensor(feats, coordinates=ct, device='cuda')).F
  net = native.Net(model, 'cuda')
  ctx = native.Context('cuda')
  scale = float(want.abs().max())
  if model.conv1.in_channels == 1:
    got = net.forward(ctx, ct)
    assert float((got - want).abs().max()) <= 2e-5 * (1 + scale)
  got2 = net.forward(ctx, ct, feats)                     # explicit features, second call on a warm arena
  assert float((got2 - want).abs().max()) <= 2e-5 * (1 + scale)
  st = ctx.stats()
  assert st['host_reads'] == 1
  with pytest.raises(abi.DgrError):
    net.forward(ctx, ct, torch.ones(len(coords), model.conv1.in_channels + 1, device='cuda'))
  net.close(); ctx.close()


def test_pair_register_native_vs_stagewise_vs_oracle(abi, dgr):
  from oracle import pipeline as op
  d, state = dgr
  xyz0, xyz1, _ = syn.room_pair(2, n_raw=20000, extent=(1.8, 1.5, 1.25))
  T_o, taps = op.register(state, xyz0, xyz1)
  d.use_icp = False
  T_n = d.register(xyz0, xyz1)
  info_n, branch_n, ctx = dict(d.last_info), d.last_branch, d._last_ctx
  assert ctx is not None and info_n['host_reads'] == 3
  # integer taps: bit-exact against the oracle
  coords = ctx.tap('coords').cpu().numpy()
  n0, n1 = info_n['n0'], info_n['n1']
  assert n0 == len(taps['coords0']) and n1 == len(taps['coords1'])
  assert np.array_equal(coords[:n0], taps['coords0'])
  c1 = coords[n0:].copy(); assert np.all(c1[:, 0] == 1); c1[:, 0] = 0
  assert np.array_equal(c1, taps['coords1'])
  sel = ctx.tap('sel').cpu().numpy()
  assert np.array_equal(sel[:n0], taps['sel0']) and np.array_equal(sel[n0:] - len(xyz0), taps['sel1'])
  assert np.array_equal(ctx.tap('xyz').cpu().numpy()[:n0], taps['xyz0'])
  F = ctx.tap('features')
  assert float((F[:n0].cpu() - taps['feat0']).abs().max()) <= 5e-5
  assert float((F[n0:].cpu() - taps['feat1']).abs().max()) <= 5e-5
  idx1 = ctx.tap('idx1').cpu().numpy()
  c6 = ctx.tap('coords6').cpu().numpy()
  assert np.array_equal(c6[:, :4], taps['coords0']) and np.array_equal(c6[:, 4:], taps['coords1'][idx1, 1:])
  # same path driven stage by stage
  T_s = d.register_stagewise(xyz0, xyz1)
  assert d.last_branch == branch_n == taps['branch']
  te, re = syn.rte_rre(T_n, T_s)        # two GPU runs differ by the atomic summation order (arg-min flips): same bar
  assert te <= 1e-3 and re <= 1e-3, (te, re)
  te, re = syn.rte_rre(T_n, T_o)
  assert te <= 1e-3 and re <= 1e-3, (te, re)
  # with ICP (the reference default), device tensors in
  d.use_icp = True
  T_i = d.register(torch.from_numpy(xyz0).cuda(), torch.from_numpy(xyz1).cuda())
  T_oi, _ = op.register(state, xyz0, xyz1, use_icp=True)
  te, re = syn.rte_rre(T_i, T_oi)
  assert te <= 1e-3 and re <= 1e-3, (te, re)
  d.use_icp = False


def test_register_stagewise_coords_feature_type_vs_oracle(abi):
  """The 'coords' inlier feature type (six input channels: cos of both points) runs stage by stage."""
  from oracle import pipeline as op
  from deepglobalregistration_b200.core.deep_global_registration import DeepGlobalRegistration
  state = syn.make_checkpoint(0, inlier_feature_type='coords')
  d = DeepGlobalRegistration(types.SimpleNamespace(weights=state, clip_weight_thresh=0.05, verbose=False))
  d.use_icp = False
  xyz0, xyz1, _ = syn.room_pair(2, n_raw=20000, extent=(1.8, 1.5, 1.25))
  T_o, taps = op.register(state, xyz0, xyz1)
  T = d.register_stagewise(xyz0, xyz1)
  assert d.last_branch == taps['branch'] == 'procrustes'
  te, re = syn.rte_rre(T, T_o)
  assert te <= 1e-3 and re <= 1e-3, (te, re)


def test_stage_methods_leave_the_taps_of_register(dgr):
  """The stage methods run on a context of their own: a call after register() keeps its taps."""
  d, _ = dgr
  xyz0, xyz1, _ = syn.room_pair(4, n_raw=15000, extent=(1.8, 1.5, 1.25))
  d.register(xyz0, xyz1)
  ctx = d._last_ctx
  sel, F = d._last_sel.clone(), ctx.tap('features')
  coords, c6 = ctx.tap('coords'), ctx.tap('coords6')
  F2 = d.fcgf_feature_extraction(torch.ones(len(coords), 1, device='cuda'), coords)
  d.inlier_prediction(torch.ones(len(c6), 1, device='cuda'), c6)
  assert d._last_ctx is ctx
  assert torch.equal(d._last_sel, sel) and torch.equal(ctx.tap('features'), F)
  assert float((F2 - F).abs().max()) <= 5e-5


def test_stage_methods_reject_malformed_input(abi, dgr):
  d, _ = dgr
  c = torch.from_numpy(_cloud(3, 500, 8, seed=3)).cuda()
  dup = torch.cat((c, c[:1]), 0)
  with pytest.raises(ValueError):
    d.fcgf_feature_extraction(torch.ones(len(dup), 1, device='cuda'), dup)
  c6 = torch.from_numpy(_cloud(6, 500, 3, seed=4)).cuda()
  dup6 = torch.cat((c6, c6[-1:]), 0)
  with pytest.raises(ValueError):
    d.inlier_prediction(torch.ones(len(dup6), 1, device='cuda'), dup6)
  with pytest.raises(abi.DgrError):
    d.fcgf_feature_extraction(torch.ones(len(c), 2, device='cuda'), c)


def test_register_batch_two_in_flight_equals_serial(dgr):
  d, _ = dgr
  pairs = [syn.room_pair(10 + i, n_raw=15000 + 1000 * i, extent=(1.8, 1.5, 1.25))[:2] for i in range(5)]
  serial = [d.register(a, b).copy() for a, b in pairs]
  batch = d.register_batch(pairs, inflight=2)
  assert len(batch) == 5
  for T_s, (T_b, branch, info) in zip(serial, batch):
    te, re = syn.rte_rre(T_b, T_s)
    assert branch == 'procrustes' and te <= 1e-3 and re <= 1e-3, (te, re)
  # float32 inputs and a lazily produced pair
  f32 = [(a.astype(np.float32), b.astype(np.float32)) for a, b in pairs[:2]]
  out = d.register_batch([f32[0], (lambda: f32[1])], inflight=2)
  assert all(o[0].shape == (4, 4) for o in out)
  st = d.native_context(0).stats()
  assert st['arena_chunks'] >= 1


def test_safeguard_branch_native_equals_stagewise(dgr):
  d, _ = dgr
  xyz0, xyz1, _ = syn.room_pair(3, n_raw=12000, extent=(1.5, 1.2, 1.0))
  keep = d.clip_weight_thresh, d.safeguard_max_iteration
  d.clip_weight_thresh, d.safeguard_max_iteration = 0.999999, 20000        # every weight clipped -> gate closed
  try:
    T_n = d.register(xyz0, xyz1)
    assert d.last_branch == 'safeguard' and d.last_info['host_reads'] == 4
    hyp, inl = d.last_info['ransac_hypothesis'], d.last_info['ransac_inliers']
    T_s = d.register_stagewise(xyz0, xyz1)
    assert d.last_branch == 'safeguard'
    # both paths evaluate the same hypotheses (counter-hash sampler); the winner can only differ when an
    # ambiguous correspondence flipped between the two feature computations (atomic summation order)
    if d.last_info['ransac_hypothesis'] == hyp:
      assert np.allclose(T_n, T_s, atol=1e-9)
    else:
      assert abs(d.last_info['ransac_inliers'] - inl) <= 3
  finally:
    d.clip_weight_thresh, d.safeguard_max_iteration = keep


@pytest.mark.parametrize('D,cin,cout,n,ext,scale', [(3, 64, 128, 5000, 10, 1.0), (3, 128, 128, 4000, 9, 1e-4),
                                                    (6, 256, 256, 3000, 3, 300.0), (3, 64, 32, 600, 5, 1.0),
                                                    (3, 192, 160, 2500, 8, 7.0)])
def test_conv_3xfp16_matches_fp32_and_3xtf32(abi, D, cin, cout, n, ext, scale):
  """The 3xFP16 mode of the tensor-core kernel against the fp32 FFMA kernel (and the 3xTF32 mode) on data of very
  different magnitudes, with heavy-tailed activations: the power-of-two scaling keeps fp16 in range."""
  from deepglobalregistration_b200.me.coords import CoordinateMapKey
  coords = _cloud(D, n, ext, seed=cin + cout)
  ct = torch.from_numpy(coords).cuda().contiguous()
  man, _, _ = _spec_and_table(abi, ct)
  _, km = man.kernel_map(CoordinateMapKey(1), 1, 3)
  g = torch.Generator().manual_seed(cin)
  nrow = len(coords)
  feat = torch.randn(nrow, cin, generator=g) * scale
  feat[::97] *= 50.0                                      # outliers set the scale; ordinary rows sit 2^5 below
  feat[1::131] *= 1e-3
  feat = feat.cuda().contiguous()
  W = (torch.randn(3 ** D, cin, cout, generator=g) / np.sqrt(cin * 8)).cuda().contiguous()
  ref64 = torch.zeros(nrow, cout, dtype=torch.float64, device='cuda')
  ii, jj = km.in_idx[:km.n_pairs].long(), km.out_idx[:km.n_pairs].long()
  kofs = km.kofs_host
  for kap in range(3 ** D):
    a, b = int(kofs[kap]), int(kofs[kap + 1])
    if b > a:
      ref64.index_add_(0, jj[a:b], feat[ii[a:b]].double() @ W[kap].double())
  out16 = abi.spconv_tc_f16_fwd(feat, W, km, torch.zeros(nrow, cout, device='cuda'))
  out32 = abi.spconv_tc_fwd(feat, abi.pack_weight_tf32(W, 3 ** D, cin, cout), km, torch.zeros(nrow, cout, device='cuda'),
                            passes=3)
  torch.cuda.synchronize()
  mag = float(ref64.abs().max())
  e16 = float((out16.double() - ref64).abs().max()) / mag
  e32 = float((out32.double() - ref64).abs().max()) / mag
  print(f'D={D} {cin}->{cout} scale {scale}: 3xFP16 err {e16:.2e}, 3xTF32 err {e32:.2e} (relative to max |out|)')
  assert e16 <= 2e-6 and e16 <= 4 * e32 + 2e-7, (e16, e32)


def test_conv1_from_occupancy_masks_equals_table_kernel(abi):
  """dgr_spconv_ones_bits_fwd (conv1 on the all-ones input, from the kernel map's bit masks) is bit-identical to
  the neighbour-table kernel fed with ones."""
  from deepglobalregistration_b200.me.coords import CoordinateMapKey, kernel_offsets
  coords = _cloud(3, 9000, 14, seed=77, batch2=True)
  ct = torch.from_numpy(coords).cuda().contiguous()
  man, spec, table = _spec_and_table(abi, ct)
  n = len(coords)
  for ks, cout in ((7, 32), (5, 64)):
    _, km = man.kernel_map(CoordinateMapKey(1), 1, ks)
    K = ks ** 3
    offs = kernel_offsets(ks, 3, 1, torch.device('cuda'))
    g = torch.Generator().manual_seed(ks)
    W = (torch.randn(K, 1, cout, generator=g) / np.sqrt(K)).cuda().contiguous()
    scale, shift = (1 + 0.1 * torch.randn(cout, generator=g)).cuda(), (0.1 * torch.randn(cout, generator=g)).cuda()
    want = abi.spconv_table_fwd(torch.ones(n, 1, device='cuda'), W, km, cout, scale, shift)
    words = torch.empty(2048, dtype=torch.int32, device='cuda')
    abi.call('dgr_bloom2_build', abi.ptr(table.keys), table.cap, abi.ptr(words), 2048, abi.stream())
    Wd = abi.lib().dgr_kmap_mask_words(n)
    bits = torch.empty(K * Wd, dtype=torch.int32, device='cuda')
    cnt = torch.empty(abi.lib().dgr_kmap_cnt_elems(K, n), dtype=torch.int32, device='cuda')
    kofs = torch.empty(K + 2, dtype=torch.int32, device='cuda')
    meta = torch.empty(5, dtype=torch.int32, device='cuda')
    abi.call('dgr_kmap_probe', abi.ptr(ct), n, None, 4, abi.ptr(spec), abi.ptr(table.keys), abi.ptr(table.vals), table.cap,
             abi.ptr(words), 2048, abi.ptr(offs), K, abi.ptr(bits), abi.ptr(cnt), abi.ptr(kofs), abi.ptr(meta), abi.stream())
    got = torch.empty(n, cout, device='cuda')
    abi.call('dgr_spconv_ones_bits_fwd', abi.ptr(W), cout, abi.ptr(bits), Wd, K, n, abi.ptr(scale), abi.ptr(shift),
             abi.ptr(got), abi.stream())
    torch.cuda.synchronize()
    assert int(meta[0]) == km.n_pairs
    assert torch.equal(got, want)
