"""Viewer entry point — same entry points as the reference's gui.py: an OrbitCamera rig (role of :28-74, written
from scratch) and NGPGUI(hparams, model_config, K, img_wh, poses, radius).render_cam() (:77-145).  The Taichi GGUI window
(Vulkan) is out of scope (SURVEY.md §2.1 row 3): render() drives the same per-frame path headlessly
along an orbit and writes PNG frames instead of presenting them."""
import os
import time
import warnings

import numpy as np
import torch

from datasets.ray_utils import get_ray_directions, get_rays
from modules.networks import MODEL_DICT
from modules.rendering import render
from modules.utils import depth2img

warnings.filterwarnings("ignore")


def _axis_angle(axis, angle):
    """Rotation by ``angle`` radians about ``axis`` (Rodrigues; the reference goes through scipy's Rotation)."""
    n = float(np.linalg.norm(axis))
    if n < 1e-12 or angle == 0.0:
        return np.eye(3)
    x, y, z = np.asarray(axis, dtype=np.float64) / n
    c, s = np.cos(angle), np.sin(angle)
    C = 1.0 - c
    return np.array([[c + x * x * C, x * y * C - z * s, x * z * C + y * s],
                     [y * x * C + z * s, c + y * y * C, y * z * C - x * s],
                     [z * x * C - y * s, z * y * C + x * s, c + z * z * C]])


class OrbitCamera:
    """Camera rig of the viewer (role of the reference's gui.py:28-74): an orientation, a look-at offset and an
    orbit distance; ``pose`` is the 4x4 camera-to-world matrix render_cam() consumes.  The camera sits ``distance``
    behind the pivot along its own viewing axis; dragging rotates about the camera's current up / right axes, the
    wheel scales the distance geometrically, panning shifts the pivot in the camera frame."""
    DRAG_DEG_PER_UNIT = 80.0       # degrees of rotation per unit of normalised mouse travel
    ZOOM_BASE = 1.1
    PAN_GAIN = 1e-4

    def __init__(self, K, img_wh, poses, r):
        self.K = K
        self.W, self.H = img_wh
        self.distance = float(r)
        self.pivot = np.zeros(3)
        first = poses[0].detach().cpu().numpy() if torch.is_tensor(poses) else np.asarray(poses[0])
        self.home = first.copy()                    # the first training pose: initial orientation
        self.orientation = first[:3, :3].astype(np.float64).copy()

    # the rest of the viewer reads these two names
    @property
    def radius(self):
        return self.distance

    @property
    def rot(self):
        return self.orientation

    @property
    def pose(self):
        eye_in_cam = np.array([0.0, 0.0, -self.distance])        # back off along the viewing (+z) axis
        c2w = np.eye(4)
        c2w[:3, :3] = self.orientation
        c2w[:3, 3] = self.orientation @ eye_in_cam - self.pivot
        return c2w

    def reset(self, pose=None):
        self.pivot = np.zeros(3)
        self.distance = 2.0
        self.orientation = np.eye(3)
        if pose is not None:
            m = pose.detach().cpu().numpy() if torch.is_tensor(pose) else np.asarray(pose)
            self.orientation = m[:3, :3].astype(np.float64).copy()

    def orbit(self, dx, dy):
        yaw = _axis_angle(self.orientation[:, 1], np.radians(self.DRAG_DEG_PER_UNIT * dx))
        pitch = _axis_angle(self.orientation[:, 0], np.radians(-self.DRAG_DEG_PER_UNIT * dy))
        self.orientation = pitch @ yaw @ self.orientation

    def scale(self, delta):
        self.distance /= self.ZOOM_BASE ** delta

    def pan(self, dx, dy, dz=0):
        self.pivot = self.pivot + self.PAN_GAIN * (self.orientation @ np.array([dx, dy, dz], dtype=np.float64))


class NGPGUI:
    def __init__(self, hparams, model_config, K, img_wh, poses, radius=4.5):
        self.hparams = hparams
        self.model = MODEL_DICT[getattr(hparams, 'model_name', 'ngp')](**model_config).cuda()
        if getattr(hparams, 'ckpt_path', None):
            print(f"loading ckpt from: {hparams.ckpt_path}")
            self.model.load_state_dict(torch.load(hparams.ckpt_path, map_location='cuda'))
        self.poses = poses
        self.cam = OrbitCamera(K, img_wh, poses, r=radius)
        self.W, self.H = img_wh
        self.exp_step_factor = 1 / 256 if hparams.dataset_name in ['colmap', 'nerfpp'] else 0
        self.dt = 0
        self.mean_samples = 0
        self.img_mode = 0
        self._directions = None

    @torch.no_grad()
    def render_cam(self):
        """One frame through render(test_time=True) (reference: gui.py:115-145)."""
        t = time.time()
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if self._directions is None:  # the reference rebuilds the pixel grid every frame (:118-123)
                self._directions = get_ray_directions(self.cam.H, self.cam.W, self.cam.K, device='cuda')
            pose = torch.tensor(self.cam.pose[:3], dtype=torch.float32, device='cuda')
            rays_o, rays_d = get_rays(self._directions, pose)
            results = render(self.model, rays_o, rays_d, test_time=True, exp_step_factor=self.exp_step_factor)
        rgb = results["rgb"].reshape(self.H, self.W, 3)
        depth = results["depth"].reshape(self.H, self.W)
        torch.cuda.synchronize()
        self.dt = time.time() - t
        self.mean_samples = results['total_samples'] / len(rays_o)
        if self.img_mode == 0:
            return rgb
        return torch.from_numpy(depth2img(depth.cpu().numpy()).astype(np.float32) / 255.0)

    def render(self, n_frames=8, out_dir='results/gui'):
        """Headless stand-in for the GGUI loop (gui.py:174-218): orbit the camera, dump frames."""
        from PIL import Image
        os.makedirs(out_dir, exist_ok=True)
        for i in range(n_frames):
            frame = self.render_cam()
            img = (frame.float().clamp(0, 1).cpu().numpy() * 255).astype(np.uint8)
            Image.fromarray(img).save(os.path.join(out_dir, f'frame_{i:03d}.png'))
            print(f'frame {i}: {1000 * self.dt:.2f} ms, {float(self.mean_samples):.2f} samples/ray')
            self.cam.orbit(0.05, 0.0)


if __name__ == "__main__":
    from datasets import dataset_dict
    from opt import get_opts
    from train import build_model_config
    hparams = get_opts()
    dataset = dataset_dict[hparams.dataset_name](root_dir=hparams.root_dir, downsample=hparams.downsample)
    NGPGUI(hparams, build_model_config(hparams), dataset.K, dataset.img_wh, dataset.poses).render()
