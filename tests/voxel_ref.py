"""fp64 torch restatement of the voxel-grid model (VoxelGrid, DESIGN.md §6d), independent of the CUDA library:
lattice mapping, masked trilinear interpolation, the real SH basis of degree <= 2, the activations, and (through
autograd) the field gradients.

The fields are only read at the corners of the given samples, so a 256^3 field never has to exist in fp64: the
corner values are gathered (fp32 -> fp64), the model is evaluated on them, and gradients wrt the gathered values are
summed onto the nodes the batch touches."""
import math

import torch

# Real SH basis in the PlenOctree convention, from the normalisation constants themselves
SQPI = math.sqrt(math.pi)
Y00 = 1 / (2 * SQPI)
Y1 = math.sqrt(3) / (2 * SQPI)
Y2_XY = math.sqrt(15) / (2 * SQPI)
Y2_ZZ = math.sqrt(5) / (4 * SQPI)
Y2_XXYY = math.sqrt(15) / (4 * SQPI)


def node_offset(G):
    return math.ceil(G / 2) - 1


def lattice(G, radius):
    """World coordinate of node i along an axis: (i - ceil(G/2) + 1) * radius, fp64 [G]."""
    return (torch.arange(G, dtype=torch.float64) - node_offset(G)) * radius


def sh_basis(deg, d):
    """d: [N,3] unit directions (fp64) -> [N, (deg+1)^2]."""
    x, y, z = d[:, 0], d[:, 1], d[:, 2]
    cols = [torch.full_like(x, Y00)]
    if deg >= 1:
        cols += [-Y1 * y, Y1 * z, -Y1 * x]
    if deg >= 2:
        cols += [Y2_XY * x * y, -Y2_XY * y * z, Y2_ZZ * (2 * z * z - x * x - y * y), -Y2_XY * x * z,
                 Y2_XXYY * (x * x - y * y)]
    return torch.stack(cols, dim=1)


def corners(xyz, G, radius, c_min):
    """The 8 corners of each sample's cell, u = (x - c_min) / radius over floor(u), floor(u)+1 per axis (corner q:
    bit 2 -> x+1, bit 1 -> y+1, bit 0 -> z+1) -> node index [N,8] (-1 outside [0,G)^3), weight [N,8] fp64."""
    u = (xyz.double() - c_min) / radius
    fl = torch.floor(u)
    fr = u - fl
    ok = torch.isfinite(fl) & (fl >= -1) & (fl < G)
    lo = torch.where(ok, fl, torch.full_like(fl, -2)).long()
    fr = torch.where(ok, fr, torch.zeros_like(fr))
    nodes, ws = [], []
    for q in range(8):
        bits = torch.tensor([(q >> 2) & 1, (q >> 1) & 1, q & 1])
        idx = lo + bits
        ws.append(torch.where(bits.bool(), fr, 1 - fr).prod(dim=1))
        valid = ((idx >= 0) & (idx < G)).all(dim=1)
        nodes.append(torch.where(valid, (idx[:, 0] * G + idx[:, 1]) * G + idx[:, 2], torch.full_like(idx[:, 0], -1)))
    return torch.stack(nodes, 1), torch.stack(ws, 1)


def gather(field, node):
    """field [G,G,G,C] (any dtype) at node [N,8] -> fp64 [N,8,C], zero at the corners outside the grid."""
    flat = field.reshape(-1, field.shape[-1])
    vals = flat[node.clamp(min=0).to(flat.device)].double().cpu()
    return torch.where((node >= 0)[..., None], vals, torch.zeros_like(vals))


def interpolate(xyz, field, radius, c_min):
    """Trilinear interpolation of field [G,G,G,C] at world points xyz [N,3]; corners outside contribute zero."""
    node, w = corners(xyz, field.shape[0], radius, c_min)
    return (w[..., None] * gather(field, node)).sum(1)


def _model(w, vals, dirs, deg, relu_mask=None):
    D = (deg + 1) ** 2
    feats = (w[..., None] * vals).sum(1)
    d = dirs.double()
    d = d / torch.norm(d, dim=1, keepdim=True)
    z = (feats[:, :3 * D].reshape(-1, 3, D) * sh_basis(deg, d)[:, None, :]).sum(-1)
    if relu_mask is None:
        return torch.relu(feats[:, -1]), torch.sigmoid(z)
    return torch.where(relu_mask, feats[:, -1], torch.zeros_like(feats[:, -1])), torch.sigmoid(z)


def default_c_min(G, radius):
    return -node_offset(G) * radius


def forward(xyz, dirs, sh, density, radius, deg, c_min=None):
    """-> sigma [N], rgb [N,3] in fp64: ReLU(density), sigmoid(sum_k Y_k(d/|d|) sh[c*D + k])."""
    G = sh.shape[0]
    c_min = default_c_min(G, radius) if c_min is None else c_min
    node, w = corners(xyz, G, radius, c_min)
    vals = torch.cat([gather(sh, node), gather(density, node)], dim=-1)
    return _model(w, vals, dirs, deg)


def scatter(node, per_corner, U_index):
    """sum of per_corner [N,8,C] onto the touched nodes: U_index = (uniq [U], inverse [N,8]) of touched_nodes."""
    uniq, inv = U_index
    out = torch.zeros(len(uniq), per_corner.shape[-1], dtype=torch.float64)
    ok = node >= 0
    out.index_add_(0, inv[ok], per_corner[ok])
    return out


def touched_nodes(node):
    """(unique valid node indices [U], position of each corner among them [N,8] (-1 for invalid corners))."""
    uniq, inv = torch.unique(node.clamp(min=-1), return_inverse=True)
    if len(uniq) and uniq[0] == -1:
        uniq, inv = uniq[1:], inv - 1
    return uniq, inv


def grads(xyz, dirs, sh, density, radius, deg, dsigma, drgb, c_min=None, relu_mask=None):
    """dL/dsh and dL/ddensity in fp64 for L = sum(dsigma * sigma) + sum(drgb * rgb), on the nodes the batch touches:
    -> (nodes [U], dsh [U, 3D], ddensity [U, 1]).  Every other node's gradient is zero.  relu_mask (bool [N]), when
    given, replaces the ReLU's own mask (interpolated density > 0): where the fp64 density is within the fp32 error of
    zero, a kernel's backward is judged with the mask its own forward chose."""
    G = sh.shape[0]
    c_min = default_c_min(G, radius) if c_min is None else c_min
    node, w = corners(xyz, G, radius, c_min)
    vals = torch.cat([gather(sh, node), gather(density, node)], dim=-1).requires_grad_(True)
    sigma, rgb = _model(w, vals, dirs, deg, relu_mask)
    ((sigma * dsigma.double()).sum() + (rgb * drgb.double()).sum()).backward()
    g = torch.where((node >= 0)[..., None], vals.grad, torch.zeros_like(vals.grad))
    idx = touched_nodes(node)
    per_node = scatter(node, g, idx)
    return idx[0], per_node[:, :-1], per_node[:, -1:]
