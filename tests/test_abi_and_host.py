"""CPU-side checks: the C-ABI library builds, loads and exports every symbol declared in
include/dgr_b200.h (no compute calls without a GPU); the ME-shaped host API has the
surface the reference touches; product code fails loudly without CUDA."""
import ctypes
import os
import re

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope='module')
def built():
  from deepglobalregistration_b200 import build
  return build.build()


def test_library_exports_and_binds_every_declared_symbol(built):
  header = open(os.path.join(ROOT, 'include', 'dgr_b200.h')).read()
  declared = set(re.findall(r'\b(dgr_[a-z0-9_]+)\s*\(', header))
  declared -= {'dgr_keyspec_t'}
  assert len(declared) >= 25
  lib = ctypes.CDLL(built)
  missing = [s for s in sorted(declared) if not hasattr(lib, s)]
  assert not missing, missing
  from deepglobalregistration_b200 import _abi
  bound = _abi.bind(built)
  assert {s for s in declared if getattr(bound, s).argtypes is not None} == declared
  assert set(_abi.DECLARATIONS) == declared, set(_abi.DECLARATIONS) ^ declared
  assert _abi.lib().dgr_version() == 100
  assert ctypes.sizeof(_abi.KeySpec) == 4 * (2 + 3 * 8)


def test_header_binding_types(tmp_path):
  """The argtypes / restypes and constants read from include/dgr_b200.h, pinned for a few declarations; a C type
  without a fixed-width ctypes equivalent is rejected, not guessed."""
  from deepglobalregistration_b200 import _abi
  p, i32, i64, u64 = ctypes.c_void_p, ctypes.c_int32, ctypes.c_int64, ctypes.c_uint64
  f32, f64 = ctypes.c_float, ctypes.c_double
  D = _abi.DECLARATIONS
  assert D['dgr_pose_graph_optimize'] == (i32, [p, i64, p, p, p, p, p, i64, f64, f64, f64, i32, i32, f64, f64, f64,
                                                f64, i32, f64, f64, p, p, p, p, p, p])
  assert D['dgr_ransac_correspondence'] == (i32, [p, p, p, p, i64, f64, i64, u64, p, p, p])
  assert D['dgr_sigmoid_clip_sum'] == (i32, [p, i64, f32, p, p, p])
  assert D['dgr_version'] == (i32, [])
  assert D['dgr_last_error'] == (ctypes.c_char_p, [])
  assert D['dgr_ctx_stream'] == (p, [p])
  assert D['dgr_kmap_mask_words'] == (i64, [i64])
  assert _abi.POINTNET_PACKED_BYTES == 1185792 and _abi.POSE_GRAPH_MAX_EDGES == 32640
  assert _abi.read_header(_abi.HEADER)[1]['DGR_TSDF_COORD_MIN'] == -1048576
  bad = tmp_path / 'bad.h'
  bad.write_text('#include <stddef.h>\nint32_t dgr_bad(const float* x, size_t n, void* stream);\n')
  with pytest.raises(_abi.DgrError, match='dgr_bad.*size_t'):
    _abi.read_header(str(bad))


def test_sm90a_sass_present(built):
  out = os.popen(f'cuobjdump -lelf {built} 2>/dev/null').read()
  assert 'sm_90a' in out


def test_no_cpu_fallback():
  from deepglobalregistration_b200 import _abi
  with pytest.raises(_abi.DgrError):
    _abi.require_device('cpu')
  if not torch.cuda.is_available():
    from deepglobalregistration_b200 import me as ME
    with pytest.raises(Exception):
      ME.SparseTensor(torch.ones(2, 1), coordinates=torch.zeros(2, 4, dtype=torch.int32))


def test_product_never_imports_oracle():
  pkg = os.path.join(ROOT, 'deepglobalregistration_b200')
  for dp, _, files in os.walk(pkg):
    for f in files:
      if f.endswith('.py'):
        src = open(os.path.join(dp, f)).read()
        assert not re.search(r'^\s*(from|import)\s+oracle\b', src, re.M), os.path.join(dp, f)


def test_me_surface_and_state_dict_layout():
  from deepglobalregistration_b200 import shims, synthetic as syn
  ME = shims.install()
  import MinkowskiEngine
  import MinkowskiEngine.MinkowskiFunctional as MEF
  assert MinkowskiEngine is ME and callable(MEF.relu)
  for name in ('SparseTensor', 'MinkowskiNetwork', 'MinkowskiConvolution', 'MinkowskiConvolutionTranspose',
               'KernelGenerator', 'RegionType', 'MinkowskiBatchNorm', 'cat', 'MinkowskiSumPooling',
               'MinkowskiPoolingTranspose', 'MinkowskiInstanceNorm', 'MinkowskiReLU', 'MinkowskiELU'):
    assert hasattr(ME, name), name
  assert callable(ME.utils.sparse_quantize) and callable(ME.utils.batched_coordinates)
  conv = ME.MinkowskiConvolution(3, 8, kernel_size=3, stride=2, has_bias=True, dimension=3)   # 0.4 spelling
  assert conv.kernel.shape == (27, 3, 8) and conv.bias.shape == (1, 8)
  assert ME.MinkowskiConvolution(3, 8, kernel_size=1, dimension=6).kernel.shape == (3, 8)
  assert ME.MinkowskiConvolutionTranspose(4, 2, kernel_size=3, stride=2, dimension=6).kernel.shape == (729, 4, 2)
  bn = ME.MinkowskiBatchNorm(8, momentum=0.05)
  assert set(bn.state_dict()) == {'bn.weight', 'bn.bias', 'bn.running_mean', 'bn.running_var',
                                  'bn.num_batches_tracked'}
  with pytest.raises(NotImplementedError):
    ME.MinkowskiInstanceNorm(8)
  bc = ME.utils.batched_coordinates([torch.zeros(3, 3).int(), torch.ones(2, 3).int()])
  assert bc.shape == (5, 4) and bc[:, 0].tolist() == [0, 0, 0, 1, 1] and bc.dtype == torch.int32
  from deepglobalregistration_b200.model import load_model
  assert load_model('NoSuchNet') is None
  for D, cin, cout, k in ((3, 1, 32, 7), (6, 1, 1, 3)):
    m = load_model('ResUNetBN2C')(cin, cout, conv1_kernel_size=k, D=D)
    sd = syn.resunet_state_dict(0, cin, cout, k, D) if D == 3 else None
    if sd is not None:
      assert m.load_state_dict(sd).missing_keys == []
    n_par = sum(p.numel() for p in m.parameters())
    assert n_par == (8_760_384 if D == 3 else 235_926_689), n_par


def test_kernel_offsets_match_oracle():
  from deepglobalregistration_b200.me.coords import kernel_offsets
  from oracle import sparse_ops as so
  for k, D, s in ((3, 3, 1), (7, 3, 1), (5, 3, 2), (3, 6, 4)):
    assert np.array_equal(kernel_offsets(k, D, s, 'cpu').numpy(), so.kernel_offsets(k, D, s))


def test_native_layer_table_parameter_order():
  """native.network_parameters lists the 66 tensors dgr_net_create documents, in execution order, for this
  package's ResUNetBN2C (the reference's attribute names, model/resunet.py:442-596)."""
  from deepglobalregistration_b200 import native, synthetic as syn
  from deepglobalregistration_b200.model import load_model
  models = [load_model('ResUNetBN2C')(1, 32, bn_momentum=0.05, conv1_kernel_size=7, normalize_feature=True, D=3)]
  C, T = [None, 32, 64, 128, 256], [None, 64, 64, 64, 128]
  for m in models:
    m.load_state_dict(syn.resunet_state_dict(0, 1, 32, 7, 3))
    m.eval()
    ps = native.network_parameters(m)
    assert len(ps) == 66 and all(p.dtype == torch.float32 and p.is_contiguous() for p in ps)
    assert tuple(ps[0].shape) == (343, 1, 32) and tuple(ps[1].shape) == (32,) and tuple(ps[2].shape) == (32,)
    assert tuple(ps[3].shape) == (27, 32, 32)                       # block1.conv1
    assert tuple(ps[9].shape) == (27, C[1], C[2])                   # conv2 (stride 2)
    assert tuple(ps[36].shape) == (27, C[4], T[4])                  # conv4_tr
    assert tuple(ps[45].shape) == (27, C[3] + T[4], T[3])           # conv3_tr reads cat(decoder, skip)
    assert tuple(ps[63].shape) == (C[1] + T[2], T[1]) and tuple(ps[64].shape) == (T[1], 32) and tuple(ps[65].shape) == (32,)
    # folded BatchNorm: scale = weight / sqrt(var + eps)
    bn = m.norm1.bn
    assert torch.allclose(ps[1], bn.weight / torch.sqrt(bn.running_var + bn.eps))
