"""Voxel-grid model (``--model_name svox``) — the reference's VoxelGrid (modules/networks.py:382-575): same constructor
arguments and parameters (``sh_fields`` [G,G,G,3*sh_dim], ``density_fields`` [G,G,G,1], fp32), with the semantics the
reference leaves unwritten decided in DESIGN.md §6d: trilinear interpolation with out-of-grid corners masked,
sigma = ReLU(density), rgb = sigmoid(SH(d) . coefficients).  Both directions run on csrc/voxel.cu.

Deviations from the reference: the occupancy grid keeps NGP's 128^3 cascades (``grid_size`` stays 128; the field
resolution is ``field_size``), and neither the hash encoder nor the MLPs that the reference's NGP.__init__ builds are
created."""
from __future__ import annotations

import torch
from torch import nn

from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.layout import make_voxel_layout, voxel_node_offset, voxel_reg_block

from .networks import MODEL_DICT, NGP, init_occupancy_grid
from .volume_train import VolumeRenderer


class _VoxelField(torch.autograd.Function):
    """forward(xyz [N,3] world, dirs [N,3], sh_fields, density_fields, model) -> sigma [N], rgb [N,3] fp32.
    backward: dL/dsh_fields and dL/ddensity_fields only (no kernel for dL/dx or dL/dd; positions that require grad are
    refused in VoxelGrid.forward)."""

    @staticmethod
    @torch.amp.custom_fwd(device_type='cuda', cast_inputs=torch.float32)
    def forward(ctx, xyz, dirs, sh, density, model):
        sigma, rgb = ops.voxel_fwd(xyz, dirs, sh.detach(), density.detach(), model._clayout)
        ctx.model = model
        ctx.save_for_backward(xyz, dirs, sigma, rgb, sh, density)
        return sigma, rgb

    @staticmethod
    @torch.amp.custom_bwd(device_type='cuda')
    def backward(ctx, dsigma, drgb):
        xyz, dirs, sigma, rgb, sh, density = ctx.saved_tensors
        m = ctx.model
        dsigma, drgb = dsigma.float().contiguous(), drgb.float().contiguous()
        if m.grad_sink is not None:
            # fused-optimizer path: accumulate straight into the trainer's flat gradient buffer
            dsh, dden = m.grad_sink
            ops.voxel_bwd(xyz, dirs, sigma, rgb, dsigma, drgb, m._clayout, dsh, dden)
            return None, None, None, None, None
        dsh = torch.zeros_like(sh, dtype=torch.float32)
        dden = torch.zeros_like(density, dtype=torch.float32)
        ops.voxel_bwd(xyz, dirs, sigma, rgb, dsigma, drgb, m._clayout, dsh, dden)
        return None, None, dsh, dden, None


class VoxelGrid(nn.Module):

    def __init__(
            self,
            scale: float = 0.5,
            half_opt: bool = False,      # accepted as in the reference; the fields are fp32 whatever its value
            # grid configs
            sh_degree: int = 2,
            grid_size: int = 256,
            grid_radius: float = 0.0125,
            origin_sh: float = 0.,
            origin_sigma: float = 0.1,
    ):
        super().__init__()
        lay = make_voxel_layout(grid_size, grid_radius, sh_degree)   # ValueError on an unsupported degree / size
        self._layout = lay
        self._clayout = lay.as_ctypes()
        self._reg_block = voxel_reg_block(lay, scale)   # the nodes the regularisers act on (NGPTrainer voxel_reg)
        self.half_opt = half_opt
        init_occupancy_grid(self, scale)
        self.sh_degree = lay.sh_degree
        self.sh_dim = lay.sh_dim
        self.field_size = lay.grid          # the reference's VoxelGrid.grid_size; grid_size is the occupancy grid's
        self.grid_radius = grid_radius
        self.origin_sh = origin_sh
        self.origin_sigma = origin_sigma
        G = self.field_size
        self.sh_fields = nn.Parameter(torch.full((G, G, G, 3 * self.sh_dim), float(origin_sh), dtype=torch.float32))
        self.density_fields = nn.Parameter(torch.full((G, G, G, 1), float(origin_sigma), dtype=torch.float32))
        self.render_func = VolumeRenderer()
        self.grad_sink = None  # optional (dsh, ddensity) fp32 buffers the backward accumulates into (NGPTrainer)

    def lattice(self) -> torch.Tensor:
        """World coordinate of node i along any axis, fp64 [G]: (i - ceil(G/2) + 1) * grid_radius
        (networks.py:450-466)."""
        i = torch.arange(self.field_size, dtype=torch.float64)
        return (i - voxel_node_offset(self.field_size)) * self.grid_radius

    # -- network ----------------------------------------------------------------------------------
    def _fusable(self, x):
        """No fused NGP kernels apply: render() sends test-time frames to render_frame's module path."""
        return False

    def density(self, x):
        """x: (N, 3) world positions -> sigmas (N) fp32, straight from the density-only kernel (no autograd)."""
        return ops.voxel_fwd(x.detach().float().contiguous(), None, None, self.density_fields.detach(),
                             self._clayout)

    def forward(self, x, d):
        """x: (N, 3) world positions, d: (N, 3) directions -> sigmas (N), rgbs (N, 3), fp32 whatever the autocast
        state."""
        if x.requires_grad:
            raise NotImplementedError("VoxelGrid has no gradient wrt the positions; pass positions that do not "
                                      "require grad")
        return _VoxelField.apply(x.float().contiguous(), d.detach().float().contiguous(), self.sh_fields,
                                 self.density_fields, self)

    # -- occupancy grid: NGP's, unchanged (they read scale, cascades, grid_size and the buffers above) -------------
    get_all_cells = NGP.get_all_cells
    sample_uniform_and_occupied_cells = NGP.sample_uniform_and_occupied_cells
    mark_invisible_cells = NGP.mark_invisible_cells
    update_density_grid = NGP.update_density_grid
    update_density_grid_reference = NGP.update_density_grid_reference
    _density_eval = NGP._density_eval        # not _fusable: falls through to density()
    grid_seed = NGP.grid_seed


MODEL_DICT['svox'] = VoxelGrid
