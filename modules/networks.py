"""NGP model wrapper — mirrors modules/networks.py of the reference: TruncExp :18-30, NGP :33-290
(same constructor arguments, buffers and state_dict keys), MLP :293-380.

The occupancy-grid maintenance (get_all_cells, sample_uniform_and_occupied_cells,
mark_invisible_cells, update_density_grid) keeps the reference's semantics with the Taichi kernels
replaced by libngp_b200 calls and without the ti.sync() host syncs.
"""
from __future__ import annotations

import math
from typing import Callable, Optional

import torch
from torch import nn

from .rendering import NEAR_DISTANCE
from .spherical_harmonics import DirEncoder
from .utils import morton3D, morton3D_invert, packbits
from .volume_train import VolumeRenderer


class TruncExp(torch.autograd.Function):
    """exp() whose backward clamps the argument to [-15, 15] (reference networks.py:18-30)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type='cuda', cast_inputs=torch.float32)
    def forward(ctx, x):
        ctx.save_for_backward(x)
        return torch.exp(x)

    @staticmethod
    @torch.amp.custom_bwd(device_type='cuda')
    def backward(ctx, dL_dout):
        x, = ctx.saved_tensors
        return dL_dout * torch.exp(x.clamp(-15, 15))


def _grid_coords(n: int) -> torch.Tensor:
    """All integer cells of an n^3 grid as [n^3, 3] int32, enumerated like
    kornia.utils.grid.create_meshgrid3d(n, n, n, False).reshape(-1, 3) which the reference uses
    (networks.py:78-86): row (d, h, w) holds (d, w, h)."""
    r = torch.arange(n, dtype=torch.int32)
    d, h, w = torch.meshgrid(r, r, r, indexing='ij')
    return torch.stack([d, w, h], dim=-1).reshape(-1, 3).contiguous()


class NGP(nn.Module):

    def __init__(
            self,
            scale: float = 0.5,
            # position encoder config
            pos_encoder_type: str = 'hash',
            levels: int = 16,
            feature_per_level: int = 2,
            log2_T: int = 19,
            base_res: int = 16,
            max_res: int = 2048,
            half_opt: bool = False,
            # mlp config
            xyz_net_width: int = 64,
            xyz_net_depth: int = 1,
            xyz_net_out_dim: int = 16,
            rgb_net_depth: int = 2,
            rgb_net_width: int = 64,
    ):
        super().__init__()
        self.scale = scale
        self.half_opt = half_opt
        self.register_buffer('center', torch.zeros(1, 3))
        self.register_buffer('xyz_min', -torch.ones(1, 3) * scale)
        self.register_buffer('xyz_max', torch.ones(1, 3) * scale)
        self.register_buffer('half_size', (self.xyz_max - self.xyz_min) / 2)

        # cascade k covers [-2^(k-1), 2^(k-1)]^3 (networks.py:62-63)
        self.cascades = max(1 + int(math.ceil(math.log2(2 * scale))), 1)
        self.grid_size = 128
        g3 = self.grid_size ** 3
        self.register_buffer('density_bitfield', torch.zeros(self.cascades * g3 // 8, dtype=torch.uint8))
        self.register_buffer('density_grid', torch.zeros(self.cascades, g3))
        self.register_buffer('grid_coords', _grid_coords(self.grid_size))

        if pos_encoder_type == 'hash':
            if half_opt:
                from .hash_encoder_half import HashEncoder
            else:
                from .hash_encoder import HashEncoder
            self.pos_encoder = HashEncoder(max_params=2 ** log2_T, base_res=base_res, max_res=max_res,
                                           levels=levels, feature_per_level=feature_per_level)
        elif pos_encoder_type == 'triplane':
            # networks.py:101-107: levels, feature_per_level, log2_T and half_opt do not apply to the tri-plane
            from .triplane import TriPlaneEncoder
            self.pos_encoder = TriPlaneEncoder(base_res=16, max_res=max_res, levels=8, feature_per_level=4)
        else:
            raise NotImplementedError(f"pos_encoder_type={pos_encoder_type!r}")
        self.pos_encoder_type = pos_encoder_type

        self.xyz_encoder = MLP(input_dim=self.pos_encoder.out_dim, output_dim=xyz_net_out_dim,
                               net_depth=xyz_net_depth, net_width=xyz_net_width, bias_enabled=False)
        self.dir_encoder = DirEncoder()
        self.rgb_net = MLP(input_dim=self.dir_encoder.out_dim + self.xyz_encoder.output_dim, output_dim=3,
                           net_depth=rgb_net_depth, net_width=rgb_net_width, bias_enabled=False,
                           output_activation=nn.Sigmoid())
        self.render_func = VolumeRenderer()

    # -- network ----------------------------------------------------------------------------------
    def _fusable(self, x):
        """True when the stock architecture is in use, so the fused sm_90a MLP kernel applies.  Which encode kernel
        runs with it is the encoder's business (encode_world / enqueue_encode_dyn: hash or tri-plane)."""
        return (x.is_cuda and _fused_mlp_available()
                and self.pos_encoder.out_dim == 32
                and self.xyz_encoder.net_depth == 1 and self.xyz_encoder.net_width == 64
                and self.xyz_encoder.output_dim == 16
                and self.rgb_net.net_depth == 2 and self.rgb_net.net_width == 64)

    def density(self, x, return_feat=False):
        """x: (N, 3) in [-scale, scale] -> sigmas (N) [, h (N, 16)]  (networks.py:136-150)."""
        x = (x - self.xyz_min) / (self.xyz_max - self.xyz_min)
        embedding = self.pos_encoder(x)
        if not return_feat and not torch.is_grad_enabled() and self._fusable(x):
            from taichi_nerfs_b200.fused_mlp import ngp_density
            return ngp_density(self, embedding)
        h = self.xyz_encoder(embedding)
        sigmas = TruncExp.apply(h[:, 0])
        if return_feat:
            return sigmas, h
        return sigmas

    def forward(self, x, d):
        """x: (N, 3) positions, d: (N, 3) directions -> sigmas (N), rgbs (N, 3)  (networks.py:152-166)."""
        if self._fusable(x):
            from taichi_nerfs_b200.fused_mlp import ngp_mlp_forward
            xn = (x - self.xyz_min) / (self.xyz_max - self.xyz_min)
            embedding = self.pos_encoder(xn)
            return ngp_mlp_forward(self, embedding, d)
        sigmas, h = self.density(x, return_feat=True)
        d = d / torch.norm(d, dim=1, keepdim=True)
        d = self.dir_encoder((d + 1) / 2)
        rgbs = self.rgb_net(torch.cat([d, h], 1))
        return sigmas, rgbs

    # -- occupancy grid -----------------------------------------------------------------------------
    @torch.no_grad()
    def get_all_cells(self):
        """[(morton indices, coords)] * cascades for every cell (networks.py:168-179)."""
        indices = morton3D(self.grid_coords).long()
        return [(indices, self.grid_coords)] * self.cascades

    @torch.no_grad()
    def sample_uniform_and_occupied_cells(self, M, density_threshold):
        """M uniform + M occupied cells per cascade (networks.py:181-209)."""
        dev = self.density_grid.device
        cells = []
        for c in range(self.cascades):
            coords1 = torch.randint(self.grid_size, (M, 3), dtype=torch.int32, device=dev)
            indices1 = morton3D(coords1).long()
            indices2 = torch.nonzero(self.density_grid[c] > density_threshold)[:, 0]
            if len(indices2) > 0:
                pick = torch.randint(len(indices2), (M,), device=dev)
                indices2 = indices2[pick]
            coords2 = morton3D_invert(indices2.int())
            cells.append((torch.cat([indices1, indices2]), torch.cat([coords1, coords2])))
        return cells

    @torch.no_grad()
    def mark_invisible_cells(self, K, poses, img_wh, chunk=32 ** 3):
        """Cells no camera sees get density -1 (networks.py:211-253); runs once before training."""
        n_cams = poses.shape[0]
        self.count_grid = torch.zeros_like(self.density_grid)
        w2c_R = poses[:, :3, :3].transpose(1, 2)
        w2c_T = -w2c_R @ poses[:, :3, 3:]
        cells = self.get_all_cells()
        for c in range(self.cascades):
            indices, coords = cells[c]
            s = min(2 ** (c - 1), self.scale)
            half_grid_size = s / self.grid_size
            for i in range(0, len(indices), chunk):
                xyzs = coords[i:i + chunk] / (self.grid_size - 1) * 2 - 1
                xyzs_w = (xyzs * (s - half_grid_size)).T
                xyzs_c = w2c_R @ xyzs_w + w2c_T
                uvd = K @ xyzs_c
                uv = uvd[:, :2] / uvd[:, 2:]
                in_image = (uvd[:, 2] >= 0) & (uv[:, 0] >= 0) & (uv[:, 0] < img_wh[0]) & \
                           (uv[:, 1] >= 0) & (uv[:, 1] < img_wh[1])
                covered = (uvd[:, 2] >= NEAR_DISTANCE) & in_image
                count = covered.sum(0) / n_cams
                self.count_grid[c, indices[i:i + chunk]] = count
                too_near = ((uvd[:, 2] < NEAR_DISTANCE) & in_image).any(0)
                valid = (count > 0) & (~too_near)
                self.density_grid[c, indices[i:i + chunk]] = torch.where(valid, 0., -1.)

    @torch.no_grad()
    def update_density_grid(self, density_threshold, warmup=False, decay=0.95, erode=False):
        """EMA-max update of the density grid + re-pack of the bitfield (networks.py:255-290) as one fixed chain of
        launches: [occupied-cell scan] -> cell pick + jittered positions -> hash + sigma net -> scatter-max -> EMA +
        partial sums -> mean -> packbits.  No torch.nonzero / len() / .item(): nothing synchronises the host, and the
        Philox-keyed draws make the grids of all ranks identical (same seed and update counter, replicated
        parameters) without a broadcast."""
        from taichi_nerfs_b200 import ops
        grid = self.density_grid
        if not grid.is_cuda:
            raise RuntimeError("update_density_grid runs on the CUDA path only (no CPU fallback)")
        if not grid.is_contiguous():
            self.density_grid = grid = grid.contiguous()
        ws = self.__dict__.get('_grid_ws')
        if ws is None or ws.device != grid.device:
            ws = self.__dict__['_grid_ws'] = ops.grid_workspace(self.cascades, self.grid_size, grid.device)
            self.__dict__['_grid_mean'] = torch.zeros(1, device=grid.device, dtype=torch.float32)
        step = self.__dict__.get('_grid_step', 0)
        self.__dict__['_grid_step'] = step + 1
        cell_idx, xyzs_w = ops.grid_sample_cells(grid, self.scale, density_threshold, warmup, self.grid_size ** 3 // 4,
                                                 self.grid_seed, step, ws)
        densities = self._density_eval(xyzs_w)
        count = None
        if erode:
            count = self.count_grid.contiguous()
        ops.grid_update(grid, cell_idx, densities, density_threshold, decay, ws, self.__dict__['_grid_mean'],
                        self.density_bitfield, count_grid=count)

    def _density_eval(self, xyzs_w):
        """sigma at world positions for the grid update: the encoder's kernel (AABB normalisation folded into it) +
        sigma net, straight on the kernels for the stock architecture, NGP.density otherwise."""
        if not self._fusable(xyzs_w):
            return self.density(xyzs_w).float().contiguous()
        from taichi_nerfs_b200 import ops
        from taichi_nerfs_b200.fused_mlp import mlp_weights
        enc = self.pos_encoder
        aabb = self.__dict__.get('_aabb6')
        if aabb is None:
            aabb = self.__dict__['_aabb6'] = (self.xyz_min.flatten().tolist()
                                               + (self.xyz_max - self.xyz_min).flatten().tolist())
        n = xyzs_w.shape[0]
        dirs = self.__dict__.get('_unit_dirs')
        if dirs is None or dirs.shape[0] < n or dirs.device != xyzs_w.device:
            dirs = torch.zeros(n, 3, device=xyzs_w.device, dtype=torch.float32)
            dirs[:, 2] = 1.0                       # the sigma head does not depend on the direction
            self.__dict__['_unit_dirs'] = dirs
        emb = enc.encode_world(xyzs_w, aabb)
        sigmas, _ = ops.mlp_fwd(emb, dirs[:n], [w.detach() for w in mlp_weights(self)])
        return sigmas

    grid_seed = 0x6E6770      # Philox key of the occupancy-grid sampler: equal on every rank by construction

    @torch.no_grad()
    def update_density_grid_reference(self, density_threshold, warmup=False, decay=0.95, erode=False):
        """The reference's own op sequence (networks.py:255-290 with torch.randint / nonzero), kept for comparison
        in tests and benchmarks; not used by the training loop."""
        tmp = torch.zeros_like(self.density_grid)
        if warmup:
            cells = self.get_all_cells()
        else:
            cells = self.sample_uniform_and_occupied_cells(self.grid_size ** 3 // 4, density_threshold)
        for c in range(self.cascades):
            indices, coords = cells[c]
            s = min(2 ** (c - 1), self.scale)
            half_grid_size = s / self.grid_size
            xyzs_w = (coords / (self.grid_size - 1) * 2 - 1) * (s - half_grid_size)
            xyzs_w += (torch.rand_like(xyzs_w) * 2 - 1) * half_grid_size
            tmp[c, indices] = self.density(xyzs_w).float()
        if erode:
            decay = torch.clamp(decay ** (1 / self.count_grid), 0.1, 0.95)
        self.density_grid = torch.where(self.density_grid < 0, self.density_grid,
                                        torch.maximum(self.density_grid * decay, tmp))
        positive = self.density_grid > 0
        mean_density = (self.density_grid * positive).sum() / positive.sum()
        from taichi_nerfs_b200 import ops
        ops.packbits(self.density_grid.reshape(-1).contiguous(), density_threshold, self.density_bitfield,
                     mean_dev=mean_density.reshape(1))


def _fused_mlp_available() -> bool:
    try:
        from taichi_nerfs_b200 import fused_mlp
        return fused_mlp.available()
    except ImportError:
        return False


class MLP(nn.Module):
    """Bias-free-capable MLP with optional skip connection every ``skip_layer`` layers — same
    constructor, attribute names and parameter keys (hidden_layers.N.weight, output_layer.weight) as
    the reference's MLP (networks.py:293-380)."""

    def __init__(
            self,
            input_dim: int,
            output_dim: int = None,
            net_depth: int = 8,
            net_width: int = 256,
            skip_layer: int = 4,
            hidden_init: Callable = nn.init.xavier_uniform_,
            hidden_activation: Callable = nn.ReLU(),
            output_enabled: bool = True,
            output_init: Optional[Callable] = nn.init.xavier_uniform_,
            output_activation: Optional[Callable] = nn.Identity(),
            bias_enabled: bool = True,
            bias_init: Callable = nn.init.zeros_,
    ):
        super().__init__()
        self.input_dim = input_dim
        self.output_dim = output_dim
        self.net_depth = net_depth
        self.net_width = net_width
        self.skip_layer = skip_layer
        self.hidden_init = hidden_init
        self.hidden_activation = hidden_activation
        self.output_enabled = output_enabled
        self.output_init = output_init
        self.output_activation = output_activation
        self.bias_enabled = bias_enabled
        self.bias_init = bias_init

        self.hidden_layers = nn.ModuleList()
        fan_in = input_dim
        for i in range(net_depth):
            self.hidden_layers.append(nn.Linear(fan_in, net_width, bias=bias_enabled))
            fan_in = net_width + input_dim if self._is_skip(i) else net_width
        if output_enabled:
            self.output_layer = nn.Linear(fan_in, output_dim, bias=bias_enabled)
        else:
            self.output_dim = fan_in
        self.initialize()

    def _is_skip(self, i):
        return self.skip_layer is not None and i > 0 and i % self.skip_layer == 0

    def initialize(self):
        def init_linear(m, w_init):
            if isinstance(m, nn.Linear):
                if w_init is not None:
                    w_init(m.weight)
                if self.bias_enabled and self.bias_init is not None:
                    self.bias_init(m.bias)

        for layer in self.hidden_layers:
            init_linear(layer, self.hidden_init)
        if self.output_enabled:
            init_linear(self.output_layer, self.output_init)

    def forward(self, x):
        inputs = x
        for i, layer in enumerate(self.hidden_layers):
            x = self.hidden_activation(layer(x))
            if self._is_skip(i):
                x = torch.cat([x, inputs], dim=-1)
        if self.output_enabled:
            x = self.output_activation(self.output_layer(x))
        return x


MODEL_DICT = {'ngp': NGP}
