"""Depth supervision (--depth_loss_w, DESIGN.md §6h): the per-ray squared error of the rendered expected depth.

``results['depth']`` is D = sum_k w_k t_k of the training render (no background term).  ``get_rays`` leaves the
camera-frame direction (u', v', 1) unnormalised, so the marcher's t, and with it D, is z-depth in the units of the pose
translations: a sensor's z-depth image is compared with D directly.  The gradient reaches the compositing's backward
through its g_depth; the graph-captured step computes the same term inside its fused per-ray head.
"""
import torch


def depth_valid(depth_gt):
    """v: the rays whose target depth is finite and > 0 (0, negative, inf or NaN mean "no depth here")."""
    return (depth_gt > 0) & torch.isfinite(depth_gt)


def depth_loss(results, depth_gt):
    """Per ray (indexed by ray id): v (D - D^)^2.  ``w * depth_loss(results, depth_gt).mean()`` is the loss term, so it
    is normalised by the batch size, not by the number of rays with a target."""
    v = depth_valid(depth_gt)
    diff = torch.where(v, results['depth'].float() - torch.where(v, depth_gt, 0.0), 0.0)
    return diff * diff
