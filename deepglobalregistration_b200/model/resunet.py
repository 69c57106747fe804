"""The ResUNet2 family (ResUNetBN2C is the FCGF extractor at D=3 and the inlier network at
D=6) on top of the ME-shaped operator API.

Same constructor signature, attribute names (hence state-dict keys) and forward graph as
the reference's ``ResUNet2`` (model/resunet.py:419-665, blocks from
model/residual_block.py:83-134, norms from model/common.py:11-13), so a checkpoint written
by the reference loads with ``load_state_dict`` unchanged.  The layers are declared from a
table instead of the reference's spelled-out constructor.  ``forward`` is the
operator-by-operator path through the ME-shaped modules (autograd, BatchNorm calibration);
inference with fused epilogues runs the same graph on the native executor
(``native.Net``, csrc/exec.cu).
"""
import torch.nn as nn

from .. import _abi
from .. import me as ME
from ..me import MinkowskiFunctional as MEF


def conv(in_channels, out_channels, kernel_size=3, stride=1, dilation=1, has_bias=False, region_type=0,
         dimension=3):
  """Reference helper (model/residual_block.py:15-44): note it never forwards has_bias or
  dilation, so these convolutions are bias-free."""
  kg = ME.KernelGenerator(kernel_size=kernel_size, stride=stride, dilation=1, dimension=dimension)
  return ME.MinkowskiConvolution(in_channels, out_channels, kernel_size=kernel_size, stride=stride,
                                 kernel_generator=kg, dimension=dimension)


def conv_tr(in_channels, out_channels, kernel_size, stride=1, dilation=1, has_bias=False,
            region_type=ME.RegionType.HYPER_CUBE, dimension=-1):
  assert dimension > 0, 'Dimension must be a positive integer'
  kg = ME.KernelGenerator(kernel_size, stride, dilation, is_transpose=True, dimension=dimension)
  return ME.MinkowskiConvolutionTranspose(in_channels=in_channels, out_channels=out_channels,
                                          kernel_size=kernel_size, stride=stride, dilation=dilation,
                                          bias=has_bias, kernel_generator=kg, dimension=dimension)


def get_norm(norm_type, num_feats, bn_momentum=0.05, dimension=-1):
  if norm_type == 'BN':
    return ME.MinkowskiBatchNorm(num_feats, momentum=bn_momentum)
  raise ValueError(f'Type {norm_type}, not defined (dgr_b200 builds BN only)')


class BasicBlockBN(nn.Module):
  """conv3-BN-ReLU-conv3-BN, add the input, ReLU (model/residual_block.py:83-134)."""

  def __init__(self, inplanes, planes, bn_momentum=0.1, D=3):
    super().__init__()
    self.conv1 = conv(inplanes, planes, kernel_size=3, stride=1, dimension=D)
    self.norm1 = get_norm('BN', planes, bn_momentum=bn_momentum, dimension=D)
    self.conv2 = conv(planes, planes, kernel_size=3, stride=1, dimension=D)
    self.norm2 = get_norm('BN', planes, bn_momentum=bn_momentum, dimension=D)

  def forward(self, x):
    out = MEF.relu(self.norm1(self.conv1(x)))
    out = self.norm2(self.conv2(out))
    out += x
    return MEF.relu(out)


class ResUNet2(ME.MinkowskiNetwork):
  NORM_TYPE = None
  BLOCK_NORM_TYPE = 'BN'
  CHANNELS = [None, 32, 64, 128, 256]
  TR_CHANNELS = [None, 32, 64, 64, 128]
  REGION_TYPE = ME.RegionType.HYPER_CUBE

  def __init__(self, in_channels=3, out_channels=32, bn_momentum=0.1, conv1_kernel_size=3,
               normalize_feature=False, D=3):
    super().__init__(D)
    C, T = self.CHANNELS, self.TR_CHANNELS
    if self.NORM_TYPE != 'BN':
      raise NotImplementedError('only the BN variants of ResUNet2 are built (released DGR weights use '
                                'ResUNetBN2C)')
    self.normalize_feature = normalize_feature
    self.conv1_kernel_size = conv1_kernel_size
    # encoder: conv{l} (stride 2 from level 2 on) -> norm{l} -> block{l}
    enc_in = [None, in_channels, C[1], C[2], C[3]]
    for l in (1, 2, 3, 4):
      k, s = (conv1_kernel_size, 1) if l == 1 else (3, 2)
      setattr(self, f'conv{l}', conv(enc_in[l], C[l], kernel_size=k, stride=s, dimension=D))
      setattr(self, f'norm{l}', get_norm(self.NORM_TYPE, C[l], bn_momentum=bn_momentum, dimension=D))
      setattr(self, f'block{l}', BasicBlockBN(C[l], C[l], bn_momentum=bn_momentum, D=D))
    # decoder: conv{l}_tr (stride 2) -> norm{l}_tr -> block{l}_tr, then concat with the skip
    dec_in = {4: C[4], 3: C[3] + T[4], 2: C[2] + T[3]}
    for l in (4, 3, 2):
      setattr(self, f'conv{l}_tr', conv_tr(dec_in[l], T[l], kernel_size=3, stride=2, dimension=D))
      setattr(self, f'norm{l}_tr', get_norm(self.NORM_TYPE, T[l], bn_momentum=bn_momentum, dimension=D))
      setattr(self, f'block{l}_tr', BasicBlockBN(T[l], T[l], bn_momentum=bn_momentum, D=D))
    self.conv1_tr = conv(C[1] + T[2], T[1], kernel_size=1, stride=1, dimension=D)
    self.final = ME.MinkowskiConvolution(T[1], out_channels, kernel_size=1, stride=1, dilation=1,
                                         bias=True, dimension=D)

  # ---------------------------------------------------------------------------------------
  def forward(self, x):
    """Operator-by-operator execution, one ME-shaped call per reference line
    (model/resunet.py:598-649)."""
    skips = {}
    out = x
    for l in (1, 2, 3, 4):
      out = getattr(self, f'conv{l}')(out)
      out = getattr(self, f'norm{l}')(out)
      out = getattr(self, f'block{l}')(out)
      skips[l] = out
      out = MEF.relu(out)
    for l in (4, 3, 2):
      out = getattr(self, f'conv{l}_tr')(out)
      out = getattr(self, f'norm{l}_tr')(out)
      out = getattr(self, f'block{l}_tr')(out)
      out = ME.cat(MEF.relu(out), skips[l - 1])
    out = MEF.relu(self.conv1_tr(out))
    out = self.final(out)
    if self.normalize_feature:
      return ME.SparseTensor(_abi.l2_normalize(out.F), coordinate_map_key=out.coordinate_map_key,
                             coordinate_manager=out.coordinate_manager)
    return out


class ResUNetBN2(ResUNet2):
  NORM_TYPE = 'BN'


class ResUNetBN2B(ResUNet2):
  NORM_TYPE = 'BN'
  TR_CHANNELS = [None, 64, 64, 64, 64]


class ResUNetBN2C(ResUNet2):
  NORM_TYPE = 'BN'
  TR_CHANNELS = [None, 64, 64, 64, 128]


class ResUNetBN2D(ResUNet2):
  NORM_TYPE = 'BN'
  TR_CHANNELS = [None, 64, 64, 128, 128]


class ResUNetBN2E(ResUNet2):
  NORM_TYPE = 'BN'
  CHANNELS = [None, 128, 128, 128, 256]
  TR_CHANNELS = [None, 64, 128, 128, 128]


class ResUNetBN2F(ResUNet2):
  NORM_TYPE = 'BN'
  CHANNELS = [None, 16, 32, 64, 128]
  TR_CHANNELS = [None, 16, 32, 64, 128]
