""""PSNR vs ref" protocol (BASELINE.json metric, SURVEY.md §8c): train the stock model on views of the reference's
shipped trained Lego model (the teacher, datasets/teacher.py) and evaluate on held-out teacher views exactly like
the reference's test loop (train.py:237-304: render(test_time=True) per view, PSNR = -10 log10(MSE), averaged).

The reference publishes 35.0 dB on the real Lego test set after 20 k steps (README.md:33-37); that dataset is not
available offline, so the number reported here is PSNR against the teacher's own renderings — it measures that the
whole CUDA training path (sampling, marching, encoding, MLP, compositing, backward, Adam, occupancy updates) learns
a real scene, not parity with the published figure.
"""
from __future__ import annotations

import time

import torch
import torch.nn.functional as F

DENSITY_THRESHOLD = 0.01 * 1024 / 3 ** 0.5   # train.py:180


def train_vs_teacher(device, steps: int = 3000, batch: int = 8192, train_views: int = 48, test_views: int = 4,
                     downsample: float = 0.5, seed: int = 23, half_opt: bool = True, graph: bool = True,
                     teacher=None, log=None, pos_encoder_type: str = 'hash'):
    """pos_encoder_type='triplane' trains the reference's tri-plane model instead (fp32 planes: half_opt does not
    apply and the loss scale is 2**19, as train.py without --half_opt; the graph-captured step is hash-only, so pass
    graph=False).  Returns {"psnr": mean dB over the held-out views, "psnr_views": [...], "steps": ..., "steps_per_s": ...,
    "rays_per_s": ..., "model": the trained NGP} or None when the teacher fixture is not staged."""
    from datasets.ray_utils import get_rays
    from datasets.teacher import TeacherLego, load_teacher
    from modules.networks import NGP
    from modules.rendering import render
    from .fast_step import StaticTrainStep
    from .trainer import NGPTrainer

    teacher = teacher if teacher is not None else load_teacher(device)
    if teacher is None:
        return None
    train_ds = TeacherLego(n_images=train_views, split='train', downsample=downsample, batch_size=batch,
                           seed=seed).to(device)
    train_ds.build_image_bank(teacher)
    test_ds = TeacherLego(n_images=test_views, split='test', downsample=downsample, seed=seed).to(device)
    test_ds.build_image_bank(teacher)

    torch.manual_seed(seed)
    if pos_encoder_type == 'triplane':
        half_opt = False
    model = NGP(scale=0.5, max_res=1024, half_opt=half_opt, pos_encoder_type=pos_encoder_type).to(device)
    model.mark_invisible_cells(train_ds.K, train_ds.poses, train_ds.img_wh)
    trainer = NGPTrainer(model, lr=1e-2, max_steps=steps)
    fast = None
    if graph:
        fast = StaticTrainStep(trainer, batch, samples_per_ray_capacity=384)
        fast.attach_ray_source(train_ds.rays, train_ds.poses, train_ds.directions, seed=seed)
    torch.cuda.synchronize(device)
    t0 = time.perf_counter()
    for step in range(steps):
        if step % 16 == 0:       # train.py:178-182
            if fast is not None:
                fast.flush()
            with torch.autocast('cuda', dtype=torch.float16):
                model.update_density_grid(DENSITY_THRESHOLD, warmup=step < 256)
        if fast is not None:
            loss = fast.step_sampled()
        else:
            b = train_ds[step]
            rays_o, rays_d = get_rays(b['direction'], b['pose'])
            loss, _ = trainer.step(rays_o, rays_d, b['rgb'])
        if log is not None and step % 500 == 0:
            log(f"step {step}: loss {float(loss):.5f}")
    if fast is not None:
        fast.flush()
    torch.cuda.synchronize(device)
    dt = time.perf_counter() - t0

    model.eval()
    psnrs = []
    with torch.no_grad():
        for i in range(len(test_ds)):
            td = test_ds[i]
            rays_o, rays_d = get_rays(test_ds.directions, td['pose'])
            with torch.autocast('cuda', dtype=torch.float16):
                res = render(model, rays_o, rays_d, test_time=True)
            mse = F.mse_loss(res['rgb'].float().clamp(0, 1), td['rgb'])
            psnrs.append(float(-10.0 * torch.log10(mse)))
    w, h = train_ds.img_wh
    return {"psnr": sum(psnrs) / len(psnrs), "psnr_views": psnrs, "steps": steps, "batch": batch,
            "train_views": train_views, "test_views": test_views, "image_wh": [w, h],
            "steps_per_s": steps / dt, "rays_per_s": steps * batch / dt, "train_seconds": dt,
            "path": "graph" if graph else "modules", "model": model, "test_dataset": test_ds}
