"""PNG codec and triangle-mesh PLY writer of io.py (CPU)."""
import zlib

import numpy as np
import pytest

from deepglobalregistration_b200 import io as dio


def _images(seed=0):
  rng = np.random.default_rng(seed)
  rgb = rng.integers(0, 256, size=(23, 37, 3), dtype=np.uint8)
  rgb[5:9] = 200                                      # flat runs as well as noise
  depth = rng.integers(0, 65536, size=(19, 41), dtype=np.uint16)
  depth[:, :7] = 1234
  return rgb, depth


@pytest.mark.parametrize('filter_type', range(5))
def test_png_round_trip(tmp_path, filter_type):
  rgb, depth = _images(filter_type)
  for name, img in (('c.png', rgb), ('d.png', depth)):
    dio.write_png(str(tmp_path / name), img, filter_type=filter_type)
    back = dio.read_png(str(tmp_path / name))
    assert back.dtype == img.dtype and back.shape == img.shape
    assert np.array_equal(back, img)
  im = dio.read_image(str(tmp_path / 'c.png'))
  assert np.array_equal(np.asarray(im), rgb)
  assert tuple(im.get_max_bound()) == (37.0, 23.0)


def test_png_against_pil(tmp_path):
  Image = pytest.importorskip('PIL.Image')
  rgb, depth = _images(7)
  dio.write_png(str(tmp_path / 'c.png'), rgb, filter_type=4)
  dio.write_png(str(tmp_path / 'd.png'), depth, filter_type=3)
  assert np.array_equal(np.asarray(Image.open(tmp_path / 'c.png').convert('RGB')), rgb)
  assert np.array_equal(np.asarray(Image.open(tmp_path / 'd.png')).astype(np.uint16), depth)
  # and files PIL writes (its own filter choice) read back
  Image.fromarray(rgb).save(tmp_path / 'pc.png')
  Image.fromarray(depth).save(tmp_path / 'pd.png')
  assert np.array_equal(dio.read_png(str(tmp_path / 'pc.png')), rgb)
  assert np.array_equal(dio.read_png(str(tmp_path / 'pd.png')), depth)


def _chunk(kind, payload):
  return len(payload).to_bytes(4, 'big') + kind + payload + zlib.crc32(kind + payload).to_bytes(4, 'big')


def test_malformed_png_raises(tmp_path):
  rgb, _ = _images(1)
  good = tmp_path / 'g.png'
  dio.write_png(str(good), rgb)
  buf = good.read_bytes()
  cases = {
      'signature': b'\x00' + buf[1:],
      'crc': buf[:40] + bytes([buf[40] ^ 0xFF]) + buf[41:],
      'truncated': buf[:len(buf) // 2],
      'no_iend': buf[:-12],
  }
  W, H = 4, 3
  rows = b''.join(b'\x00' + bytes(W * 4) for _ in range(H))
  rgba = dio._PNG_SIG + _chunk(b'IHDR', W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([8, 6, 0, 0, 0])) + \
      _chunk(b'IDAT', zlib.compress(rows)) + _chunk(b'IEND', b'')
  cases['rgba'] = rgba
  inter = dio._PNG_SIG + _chunk(b'IHDR', W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([8, 2, 0, 0, 1])) + \
      _chunk(b'IDAT', zlib.compress(b''.join(b'\x00' + bytes(W * 3) for _ in range(H)))) + _chunk(b'IEND', b'')
  cases['interlaced'] = inter
  badf = dio._PNG_SIG + _chunk(b'IHDR', W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([8, 2, 0, 0, 0])) + \
      _chunk(b'IDAT', zlib.compress(b''.join(b'\x07' + bytes(W * 3) for _ in range(H)))) + _chunk(b'IEND', b'')
  cases['filter'] = badf
  short = dio._PNG_SIG + _chunk(b'IHDR', W.to_bytes(4, 'big') + H.to_bytes(4, 'big') + bytes([8, 2, 0, 0, 0])) + \
      _chunk(b'IDAT', zlib.compress(bytes(5))) + _chunk(b'IEND', b'')
  cases['short_data'] = short
  for name, data in cases.items():
    p = tmp_path / f'{name}.png'
    p.write_bytes(data)
    with pytest.raises(ValueError):
      dio.read_png(str(p))
  with pytest.raises(ValueError):
    dio.write_png(str(tmp_path / 'x.png'), np.zeros((4, 4), np.uint8))


def test_mesh_ply_round_trip(tmp_path):
  rng = np.random.default_rng(3)
  V = rng.normal(size=(50, 3))
  T = rng.integers(0, 50, size=(80, 3)).astype(np.int32)
  C = rng.uniform(0, 1, size=(50, 3))
  mesh = dio.TriangleMesh(V, T, C)
  assert dio.write_triangle_mesh(str(tmp_path / 'm.ply'), mesh)
  pc = dio.read_point_cloud(str(tmp_path / 'm.ply'))
  assert np.array_equal(pc.points, V.astype(np.float32).astype(np.float64))
  _, extra = dio.read_ply(str(tmp_path / 'm.ply'))
  assert np.array_equal(extra['red'], np.round(C[:, 0] * 255).astype(np.uint8))
  # the face element follows the vertices: parse it back
  buf = (tmp_path / 'm.ply').read_bytes()
  body = buf[buf.index(b'end_header\n') + len(b'end_header\n'):]
  faces = np.frombuffer(body[50 * 15:], dtype=[('n', 'u1'), ('v', '<i4', (3,))])
  assert (faces['n'] == 3).all() and np.array_equal(faces['v'], T)
  # without colours, and empty
  dio.write_triangle_mesh(str(tmp_path / 'n.ply'), dio.TriangleMesh(V, T))
  assert np.array_equal(dio.read_point_cloud(str(tmp_path / 'n.ply')).points, V.astype(np.float32))
  dio.write_triangle_mesh(str(tmp_path / 'e.ply'), dio.TriangleMesh())
  assert dio.read_point_cloud(str(tmp_path / 'e.ply')).points.shape == (0, 3)
  with pytest.raises(ValueError):
    dio.write_triangle_mesh(str(tmp_path / 'bad.ply'), dio.TriangleMesh(V, T + 50))
