"""Reader for COLMAP's binary sparse model (``sparse/0/{cameras,images,points3D}.bin``), written from the format
COLMAP documents (src/base/reconstruction.cc, Read*Binary): little-endian, counts as uint64.

    cameras.bin   u64 n; n x (i32 camera_id, i32 model_id, u64 width, u64 height, f64 params[num_params(model)])
    images.bin    u64 n; n x (i32 image_id, f64 qvec[4] (w, x, y, z), f64 tvec[3], i32 camera_id,
                              name (bytes up to a NUL), u64 n2d, n2d x (f64 x, f64 y, i64 point3D_id))
    points3D.bin  u64 n; n x (u64 point3D_id, f64 xyz[3], u8 rgb[3], f64 error,
                              u64 track_length, track_length x (i32 image_id, i32 point2D_idx))

Each reader returns a dict keyed by id in file order, as the reference's colmap_utils.py does (its ColmapDataset
depends on that order, colmap.py:49-68).  A file that ends inside a record, or a camera model id COLMAP does not
define, raises ``ValueError`` instead of reading past the end.
"""
from __future__ import annotations

import struct
from typing import NamedTuple

import numpy as np

# model id -> (name, number of parameters); COLMAP's camera model table (src/base/camera_models.h)
CAMERA_MODELS = {
    0: ('SIMPLE_PINHOLE', 3), 1: ('PINHOLE', 4), 2: ('SIMPLE_RADIAL', 4), 3: ('RADIAL', 5), 4: ('OPENCV', 8),
    5: ('OPENCV_FISHEYE', 8), 6: ('FULL_OPENCV', 12), 7: ('FOV', 5), 8: ('SIMPLE_RADIAL_FISHEYE', 4),
    9: ('RADIAL_FISHEYE', 5), 10: ('THIN_PRISM_FISHEYE', 12),
}


class Camera(NamedTuple):
    id: int
    model: str
    width: int
    height: int
    params: np.ndarray          # float64


class Image(NamedTuple):
    id: int
    qvec: np.ndarray            # float64 (w, x, y, z): world-to-camera rotation
    tvec: np.ndarray            # float64: world-to-camera translation
    camera_id: int
    name: str
    xys: np.ndarray             # [n2d, 2] float64
    point3D_ids: np.ndarray     # [n2d] int64

    def qvec2rotmat(self):
        return qvec2rotmat(self.qvec)


class Point3D(NamedTuple):
    id: int
    xyz: np.ndarray             # float64
    rgb: np.ndarray             # uint8
    error: float
    image_ids: np.ndarray       # int32
    point2D_idxs: np.ndarray    # int32


def qvec2rotmat(qvec):
    """Rotation matrix of the unit quaternion (w, x, y, z), in the reference's operation order
    (colmap_utils.py:301-316) so that poses come out bit-identical."""
    w, x, y, z = qvec
    return np.array([[1 - 2 * y**2 - 2 * z**2, 2 * x * y - 2 * w * z, 2 * z * x + 2 * w * y],
                     [2 * x * y + 2 * w * z, 1 - 2 * x**2 - 2 * z**2, 2 * y * z - 2 * w * x],
                     [2 * z * x - 2 * w * y, 2 * y * z + 2 * w * x, 1 - 2 * x**2 - 2 * y**2]])


class _Reader:
    def __init__(self, path):
        self.path = path
        with open(path, 'rb') as f:
            self.buf = f.read()
        self.pos = 0

    def take(self, n):
        if n < 0 or self.pos + n > len(self.buf):
            raise ValueError(f"{self.path}: truncated ({len(self.buf)} bytes, a record needs bytes up to "
                             f"{self.pos + n})")
        out = self.buf[self.pos:self.pos + n]
        self.pos += n
        return out

    def unpack(self, fmt):
        return struct.unpack('<' + fmt, self.take(struct.calcsize('<' + fmt)))

    def array(self, dtype, count):
        dt = np.dtype(dtype).newbyteorder('<')
        return np.frombuffer(self.take(dt.itemsize * count), dtype=dt).astype(dtype)

    def cstring(self):
        end = self.buf.find(b'\0', self.pos)
        if end < 0:
            raise ValueError(f"{self.path}: truncated (image name without its terminating NUL)")
        s = self.buf[self.pos:end].decode('utf-8')
        self.pos = end + 1
        return s

    def count(self, record_bytes):
        """A u64 record count, refused when even the smallest records would not fit in the rest of the file."""
        n, = self.unpack('Q')
        if n * record_bytes > len(self.buf) - self.pos:
            raise ValueError(f"{self.path}: truncated ({n} records cannot fit in {len(self.buf) - self.pos} bytes)")
        return n

    def done(self):
        if self.pos != len(self.buf):
            raise ValueError(f"{self.path}: {len(self.buf) - self.pos} trailing bytes after the last record")


def read_cameras_binary(path):
    r = _Reader(path)
    cams = {}
    for _ in range(r.count(24)):
        cam_id, model_id, width, height = r.unpack('iiQQ')
        if model_id not in CAMERA_MODELS:
            raise ValueError(f"{path}: camera {cam_id} has model id {model_id}, which COLMAP does not define")
        name, n_params = CAMERA_MODELS[model_id]
        cams[cam_id] = Camera(cam_id, name, width, height, np.array(r.unpack('d' * n_params)))
    r.done()
    return cams


def read_images_binary(path):
    r = _Reader(path)
    imgs = {}
    for _ in range(r.count(73)):
        props = r.unpack('idddddddi')
        img_id, qvec, tvec, cam_id = props[0], np.array(props[1:5]), np.array(props[5:8]), props[8]
        name = r.cstring()
        n2d, = r.unpack('Q')
        rec = np.frombuffer(r.take(24 * n2d), dtype=np.dtype([('x', '<f8'), ('y', '<f8'), ('id', '<i8')]))
        xys = np.stack([rec['x'], rec['y']], 1).astype(np.float64)
        imgs[img_id] = Image(img_id, qvec, tvec, cam_id, name, xys, rec['id'].astype(np.int64))
    r.done()
    return imgs


def read_points3d_binary(path):
    r = _Reader(path)
    pts = {}
    for _ in range(r.count(51)):
        props = r.unpack('QdddBBBd')
        pid, xyz, rgb, err = props[0], np.array(props[1:4]), np.array(props[4:7], dtype=np.uint8), props[7]
        track_len, = r.unpack('Q')
        track = r.array(np.int32, 2 * track_len).reshape(-1, 2)
        pts[pid] = Point3D(pid, xyz, rgb, err, track[:, 0].copy(), track[:, 1].copy())
    r.done()
    return pts
