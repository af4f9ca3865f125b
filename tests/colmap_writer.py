"""Writes COLMAP binary sparse models (the layout datasets/colmap_model.py documents): the fixture generator
uses it for tests/golden/datasets/360_v2/, and the reader's tests round-trip through it."""
from __future__ import annotations

import os
import struct

import numpy as np

MODEL_IDS = {'SIMPLE_PINHOLE': 0, 'PINHOLE': 1, 'SIMPLE_RADIAL': 2, 'RADIAL': 3, 'OPENCV': 4, 'OPENCV_FISHEYE': 5,
             'FULL_OPENCV': 6, 'FOV': 7, 'SIMPLE_RADIAL_FISHEYE': 8, 'RADIAL_FISHEYE': 9, 'THIN_PRISM_FISHEYE': 10}


def cameras_bytes(cams):
    """cams: list of (camera_id, model name or id, width, height, params)."""
    out = [struct.pack('<Q', len(cams))]
    for cid, model, w, h, params in cams:
        mid = MODEL_IDS[model] if isinstance(model, str) else model
        out.append(struct.pack('<iiQQ', cid, mid, w, h) + struct.pack('<' + 'd' * len(params), *params))
    return b''.join(out)


def images_bytes(imgs):
    """imgs: list of (image_id, qvec (w,x,y,z), tvec, camera_id, name, xys [n,2], point3D_ids [n])."""
    out = [struct.pack('<Q', len(imgs))]
    for iid, q, t, cid, name, xys, pids in imgs:
        out.append(struct.pack('<idddddddi', iid, *q, *t, cid) + name.encode() + b'\0')
        out.append(struct.pack('<Q', len(pids)))
        for (x, y), p in zip(xys, pids):
            out.append(struct.pack('<ddq', x, y, p))
    return b''.join(out)


def points_bytes(pts):
    """pts: list of (point3D_id, xyz, rgb, error, image_ids, point2D_idxs)."""
    out = [struct.pack('<Q', len(pts))]
    for pid, xyz, rgb, err, iids, p2d in pts:
        out.append(struct.pack('<QdddBBBd', pid, *xyz, *rgb, err) + struct.pack('<Q', len(iids)))
        out.append(np.stack([np.asarray(iids, '<i4'), np.asarray(p2d, '<i4')], 1).tobytes())
    return b''.join(out)


def write_model(sparse_dir, cams, imgs, pts):
    os.makedirs(sparse_dir, exist_ok=True)
    for name, data in (('cameras.bin', cameras_bytes(cams)), ('images.bin', images_bytes(imgs)),
                       ('points3D.bin', points_bytes(pts))):
        with open(os.path.join(sparse_dir, name), 'wb') as f:
            f.write(data)


def rotmat2qvec(R):
    """Unit quaternion (w, x, y, z) of a rotation matrix, w >= 0."""
    tr = np.trace(R)
    w = np.sqrt(max(0.0, 1 + tr)) / 2
    x = np.copysign(np.sqrt(max(0.0, 1 + R[0, 0] - R[1, 1] - R[2, 2])) / 2, R[2, 1] - R[1, 2])
    y = np.copysign(np.sqrt(max(0.0, 1 - R[0, 0] + R[1, 1] - R[2, 2])) / 2, R[0, 2] - R[2, 0])
    z = np.copysign(np.sqrt(max(0.0, 1 - R[0, 0] - R[1, 1] + R[2, 2])) / 2, R[1, 0] - R[0, 1])
    q = np.array([w, x, y, z])
    return q / np.linalg.norm(q)
