"""Training entry point — same CLI and loop structure as the reference's train.py (main() :35-322):
seeds (:39-42), model_config (:86-117), mark_invisible_cells (:129), loss scale 2**16 | 2**19 (:137-141),
Adam(lr, eps=1e-15) + cosine annealing to lr/30 (:143-163), density-grid update every 16 steps with a
256-step warm-up (:57-58,178-182), log line every 1000 steps (:203-219), results/model.pth (:232-235),
test-split PSNR and SSIM (:237-304); with --extract_mesh, results/mesh.ply after the evaluation (DESIGN.md §6g).
With --depth_loss_w the loss gains the depth term (DESIGN.md §6h) and a test split with depth reports depth_mae.
With --extrinsics_lr every training image's pose is refined with the model (DESIGN.md §6i): the training rays come from
the corrected poses, results/poses_refined.npy holds them at the end; the test split keeps its poses as loaded.
With --ray_sampling_strategy error_map the training pixels are drawn from a per-tile error map (DESIGN.md §6j) that is
rebuilt beside every density-grid update; every per-ray loss term is weighted by the ray's weight, and
results/error_map.npy holds the map at the end.
With --exposure_lr every training image gets a learned per-channel exposure (DESIGN.md §6k) that scales its rays' sample
colours; results/exposures.npy holds them (stops) at the end, and test views render at the mean exposure, e = 0.
With --lens_distortion a COLMAP or ngp scene keeps its lens distortion and every pixel's direction is unprojected
through it; with --intrinsics_lr the training camera's focal length and principal point are refined with the model
(DESIGN.md §6l): the training rays come from the rays' pixels under the corrected intrinsics, test views render through
the refined camera, and results/intrinsics_refined.json holds it at the end.
The step body runs on the sm_90a kernels through NGPTrainer (fused Adam,
no host sync for the inf check); under torchrun every rank trains on its own rays and the gradients are summed
once per step: by the peer-memory optimizer kernel when all ranks share one NVLink box, else by an fp16 NCCL
all-reduce of the flat gradient buffer.
"""
import os
import random
import time
import warnings

import numpy as np
import torch
import torch.nn.functional as F

from datasets import dataset_dict
from datasets.ray_utils import get_rays
from modules.depth import depth_loss, depth_valid
from modules.distortion import distortion_loss
from modules.networks import MODEL_DICT
from modules.rendering import MAX_SAMPLES, render
from modules.utils import depth2img, save_deployment_model
from opt import DISK_DATASETS, get_opts
from taichi_nerfs_b200 import ops
from taichi_nerfs_b200.trainer import NGPTrainer

warnings.filterwarnings("ignore")


def build_model_config(hparams):
    if getattr(hparams, 'model_name', 'ngp') == 'svox':   # VoxelGrid's keyword arguments (networks.py:383-393)
        return {'scale': hparams.scale, 'half_opt': hparams.half_opt, 'sh_degree': hparams.sh_degree,
                'grid_size': hparams.grid_size, 'grid_radius': hparams.grid_radius, 'origin_sh': hparams.origin_sh,
                'origin_sigma': hparams.origin_sigma}
    if hparams.deployment:  # train.py:88-99
        return {'scale': hparams.scale, 'pos_encoder_type': 'hash', 'levels': 4, 'feature_per_level': 4,
                'base_res': 32, 'max_res': 128, 'log2_T': 21, 'xyz_net_width': 16, 'rgb_net_width': 16,
                'rgb_net_depth': 1}
    return {'scale': hparams.scale, 'pos_encoder_type': hparams.encoder_type,
            'max_res': 1024 if hparams.scale == 0.5 else 4096, 'half_opt': hparams.half_opt}


def save_mesh(model, hparams, path):
    """Marching cubes of the model's density lattice (--mesh_res, --mesh_threshold, --mesh_bound) written as PLY."""
    from taichi_nerfs_b200.mesh import extract_mesh, write_ply
    mesh = extract_mesh(model, hparams.mesh_res, hparams.mesh_threshold, hparams.mesh_bound)
    write_ply(path, mesh)
    print(f"mesh: {len(mesh.vertices)} vertices, {len(mesh.faces)} faces -> {path}")


def psnr_of(mse):
    return -10.0 * torch.log10(mse)


def main(prefix_args=None):
    hparams = get_opts(prefix_args)
    world = int(os.environ.get("WORLD_SIZE", "1"))
    rank = int(os.environ.get("RANK", "0"))
    local = int(os.environ.get("LOCAL_RANK", str(max(hparams.gpu, 0))))
    if not torch.cuda.is_available():
        raise RuntimeError("train.py needs a CUDA device: the hot path has no CPU fallback")
    device = torch.device("cuda", local)
    torch.cuda.set_device(device)
    if world > 1 and hparams.ray_sampling_strategy == 'error_map':
        raise ValueError("--ray_sampling_strategy error_map trains on one GPU: the error map is not shared between ranks")
    if world > 1 and hparams.extrinsics_lr > 0:
        raise ValueError("--extrinsics_lr trains on one GPU: the pose gradient is not exchanged between ranks")
    if world > 1 and hparams.intrinsics_lr > 0:
        raise ValueError("--intrinsics_lr trains on one GPU: the intrinsics gradient is not exchanged between ranks")
    if world > 1 and hparams.exposure_lr > 0:
        raise ValueError("--exposure_lr trains on one GPU: the exposure gradient is not exchanged between ranks")
    if world > 1:
        torch.distributed.init_process_group("nccl", device_id=device)

    seed = 23
    random.seed(seed + rank)
    np.random.seed(seed + rank)
    torch.manual_seed(seed)  # same parameter init on every rank

    val_dir = 'results/'
    exp_step_factor = 1 / 256 if hparams.scale > 0.5 else 0.
    warmup_steps, update_interval = 256, 16

    dataset = dataset_dict[hparams.dataset_name]
    if hparams.dataset_name in DISK_DATASETS:   # the reference's arguments only (train.py:61-73)
        extra = {'lens_distortion': True} if hparams.lens_distortion else {}
        train_dataset = dataset(root_dir=hparams.root_dir, split=hparams.split,
                                downsample=hparams.downsample, **extra).to(device)
        test_dataset = dataset(root_dir=hparams.root_dir, split='test', downsample=hparams.downsample,
                               **extra).to(device)
    else:
        extra = {'scene': 'analytic'} if hparams.dataset_name == 'synthetic' else {}
        if hparams.depth_loss_w > 0:
            extra['with_depth'] = True
        train_dataset = dataset(root_dir=hparams.root_dir, split=hparams.split, downsample=hparams.downsample,
                                seed=seed, **extra).to(device)
        train_dataset._seed = seed + rank  # different rays per rank
        test_dataset = dataset(root_dir=hparams.root_dir, split='test', downsample=hparams.downsample,
                               n_images=4, **extra).to(device)
    train_dataset.batch_size = hparams.batch_size
    error_map = None
    if hparams.ray_sampling_strategy == 'error_map':   # the map draws the pixels; the dataset gathers them
        from taichi_nerfs_b200.error_map import ErrorMap
        error_map = ErrorMap(len(train_dataset.poses), *train_dataset.img_wh, res=hparams.error_map_res,
                             seed=seed + rank, device=device)
    else:
        train_dataset.ray_sampling_strategy = hparams.ray_sampling_strategy
    model_config = build_model_config(hparams)
    model = MODEL_DICT[hparams.model_name](**model_config).to(device)
    if hparams.ckpt_path:
        model.load_state_dict(torch.load(hparams.ckpt_path, map_location=device))
        print("Load checkpoint from %s" % hparams.ckpt_path)
    camera = getattr(train_dataset, 'camera', None)   # set by --lens_distortion (DESIGN.md §6l)
    if camera is not None:
        model.mark_invisible_cells(train_dataset.K, train_dataset.poses, train_dataset.img_wh, camera=camera)
    else:
        model.mark_invisible_cells(train_dataset.K, train_dataset.poses, train_dataset.img_wh)

    torch.manual_seed(seed + rank)  # data / marching noise differ per rank from here on
    voxel_reg = None
    if hparams.model_name == 'svox':   # total variation / sparsity weights; all 0 (the default) enqueue nothing
        voxel_reg = (hparams.tv_sigma_loss_w, hparams.tv_sh_loss_w, hparams.sparsity_loss_w)
    extrinsics = None
    if hparams.extrinsics_lr > 0:   # per-image pose corrections (DESIGN.md §6i)
        from taichi_nerfs_b200.extrinsics import PoseRefinement
        extrinsics = PoseRefinement(train_dataset.poses, hparams.extrinsics_lr / hparams.lr)
    intrinsics = None
    if hparams.intrinsics_lr > 0:   # the training camera's focal length and principal point (DESIGN.md §6l)
        from taichi_nerfs_b200.intrinsics import Camera, IntrinsicsRefinement
        if camera is None:
            K = train_dataset.K.double().cpu()
            camera = Camera('PINHOLE', float(K[0, 0]), float(K[1, 1]), float(K[0, 2]), float(K[1, 2]))
        intrinsics = IntrinsicsRefinement(camera, *train_dataset.img_wh, hparams.intrinsics_lr / hparams.lr,
                                          train_dataset.poses)
    exposure = None
    if hparams.exposure_lr > 0:   # per-image exposures (DESIGN.md §6k)
        from taichi_nerfs_b200.exposure import ExposureCorrection
        exposure = ExposureCorrection(len(train_dataset.poses), hparams.exposure_lr / hparams.lr, device)
    trainer = NGPTrainer(model, lr=hparams.lr, max_steps=hparams.max_steps, voxel_reg=voxel_reg,
                         extrinsics=extrinsics, exposure=exposure, intrinsics=intrinsics)

    # --random_bg (DESIGN.md §6f): every training ray gets its own background colour, drawn on the device
    bg_load = getattr(train_dataset, 'bg_load', 1.0)
    fast = None
    if hparams.graph_step:
        if not model._fusable(next(model.parameters())):
            raise ValueError("--graph_step needs the stock NGP architecture")
        if getattr(model, 'pos_encoder_type', 'hash') != 'hash':
            raise ValueError("--graph_step runs the hash encoder only; train a tri-plane model without it")
        from taichi_nerfs_b200.fast_step import StaticTrainStep
        fast = StaticTrainStep(trainer, hparams.batch_size, exp_step_factor=exp_step_factor,
                               distortion_loss_w=hparams.distortion_loss_w, random_bg=hparams.random_bg,
                               bg_seed=seed + rank, bg_load=bg_load, depth_loss_w=hparams.depth_loss_w,
                               extrinsics=extrinsics, error_map=error_map)

    tic = time.time()
    for step in range(hparams.max_steps + 1):
        model.train()
        if error_map is None:
            data = train_dataset[step % len(train_dataset)]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if step % update_interval == 0:
                model.update_density_grid(0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=step < warmup_steps)
        ray_w = None
        if error_map is not None:
            if step % update_interval == 0 and step > 0:
                error_map.rebuild()
            em_img, em_pix, ray_w = error_map.draw(hparams.batch_size, step)
            data = train_dataset.gather(em_img, em_pix)
        img_idxs = rays_o = rays_d = pix_idxs = None
        if extrinsics is not None or exposure is not None or intrinsics is not None:
            img_idxs = torch.as_tensor(data['img_idxs'], device=device)   # same_image: one index, broadcast
        direction = data['direction']
        if intrinsics is not None:
            pix_idxs = torch.as_tensor(data['pix_idxs'], device=device)
            if fast is None:         # the graph step unprojects the pixels itself
                direction = intrinsics.directions(pix_idxs)
        if fast is not None and (extrinsics is not None or intrinsics is not None):
            pass                     # the graph step forms the rays itself
        elif extrinsics is not None:
            rays_o, rays_d = extrinsics.rays(direction, img_idxs)
        else:
            rays_o, rays_d = get_rays(direction, data['pose'])
        depth = None
        if hparams.depth_loss_w > 0:
            depth = data.get('depth')
            if depth is None:
                raise ValueError(f"--depth_loss_w: the {hparams.dataset_name} dataset at {hparams.root_dir!r} has no "
                                 f"depth (an ngp scene needs depth_path frames)")
        terms = []
        per_ray = (lambda v: v.mean()) if ray_w is None else (lambda v: (v * ray_w).mean())  # noqa: E731
        if hparams.distortion_loss_w > 0:
            terms.append(lambda res: hparams.distortion_loss_w * per_ray(distortion_loss(res)))
        if depth is not None:
            terms.append(lambda res: hparams.depth_loss_w * per_ray(depth_loss(res, depth)))
        extra_loss = (lambda res: sum(f(res) for f in terms)) if terms else None  # noqa: E731
        if fast is not None:   # one graph replay, nothing synchronises the host
            em_args = {} if error_map is None else {'ray_w': ray_w, 'img_idxs': em_img, 'pix_idxs': em_pix}
            if exposure is not None and error_map is None:
                em_args['img_idxs'] = img_idxs
            if intrinsics is not None:   # the step forms the rays from the pixels itself
                loss = fast.step(None, None, data['rgb'], alpha=data.get('alpha') if hparams.random_bg else None,
                                 depth=depth, **{**em_args, 'img_idxs': img_idxs, 'pix_idxs': pix_idxs})
            elif extrinsics is not None:   # the step forms the rays from the corrected poses itself
                loss = fast.step(None, None, data['rgb'], alpha=data.get('alpha') if hparams.random_bg else None,
                                 depth=depth, directions=data['direction'], **{'img_idxs': img_idxs, **em_args})
            else:
                loss = fast.step(rays_o, rays_d, data['rgb'],
                                 alpha=data.get('alpha') if hparams.random_bg else None, depth=depth, **em_args)
            results = {'rgb': fast.rgb, 'rm_samples': fast.counter[0].clamp(max=fast.cap), 'vr_samples':
                       fast.counter[0].clamp(max=fast.cap), 'dropped_rays': fast.counter[1]}
        else:
            bg_rgb = None
            if hparams.random_bg:   # the colours of step trainer.step_count + 1, as the graph step draws them
                bg_rgb = ops.random_bg(seed + rank, trainer.step_count + 1, len(rays_o), device)
            loss, results = trainer.step(rays_o, rays_d, data['rgb'], exp_step_factor, extra_loss=extra_loss,
                                         bg_rgb=bg_rgb, alpha=data.get('alpha'), b_load=bg_load, img_idxs=img_idxs,
                                         ray_w=ray_w, pix_idxs=pix_idxs)
            if error_map is not None:   # the graph step accumulates inside its graph
                error_map.accumulate(results['rgb'].float(), data['rgb'], em_img, em_pix, bg_rgb=bg_rgb,
                                     alpha=data.get('alpha') if bg_rgb is not None else None, b_load=bg_load)

        if step % 1000 == 0 and rank == 0:
            with torch.no_grad():
                mse = F.mse_loss(results['rgb'].float(), data['rgb'])
                n = len(data['rgb'])
                print(f"elapsed_time={time.time() - tic:.2f}s | step={step} | psnr={psnr_of(mse):.2f} | "
                      f"loss={float(loss):.6f} | rays={n} | rm_s={float(results['rm_samples']) / n:.1f} | "
                      f"vr_s={float(results['vr_samples']) / n:.1f} | "
                      + (f"rays truncated/dropped for capacity={int(results['dropped_rays'])} | "
                         if int(results.get('dropped_rays', 0)) else ""))

    if rank != 0:
        return
    if hparams.deployment:
        save_deployment_model(model=model, dataset=train_dataset, save_dir=hparams.deployment_model_path)
    os.makedirs(val_dir, exist_ok=True)
    torch.save(model.state_dict(), os.path.join(val_dir, 'model.pth'))
    if error_map is not None:
        np.save(os.path.join(val_dir, 'error_map.npy'), error_map.as_image().cpu().numpy())
    if exposure is not None:
        e = exposure.exposures()
        np.save(os.path.join(val_dir, 'exposures.npy'), e)
        print(f"exposure: mean |e| = {float(np.abs(e).mean()):.4f} stops | max |e| = {float(np.abs(e).max()):.4f} "
              f"stops -> {os.path.join(val_dir, 'exposures.npy')}")
    if intrinsics is not None:
        import json
        fx, fy, cx, cy = intrinsics.refined()
        c = intrinsics.camera
        with open(os.path.join(val_dir, 'intrinsics_refined.json'), 'w') as f:
            json.dump({**c.as_dict(), 'fx': fx, 'fy': fy, 'cx': cx, 'cy': cy}, f, indent=1)
        print(f"intrinsics: focal x{fx / c.fx:.5f} | principal point ({cx - c.cx:+.3f}, {cy - c.cy:+.3f}) px -> "
              f"{os.path.join(val_dir, 'intrinsics_refined.json')}")
    if extrinsics is not None:
        np.save(os.path.join(val_dir, 'poses_refined.npy'), extrinsics.refined_poses())
        rot_deg, trans = extrinsics.mean_correction()
        print(f"extrinsics: mean |omega| = {rot_deg:.4f} deg | mean |tau| = {trans:.6f} -> "
              f"{os.path.join(val_dir, 'poses_refined.npy')}")

    # test loop (train.py:237-304): PSNR and SSIM per held-out view; first view saved as PNG
    model.eval()
    w, h = test_dataset.img_wh
    psnrs, ssims, depth_maes = [], [], []
    # the test views share the training camera: with intrinsics refinement they render through the refined one
    test_dirs = test_dataset.directions if intrinsics is None else intrinsics.table()
    with torch.no_grad():
        for i in range(len(test_dataset)):
            td = test_dataset[i]
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                rays_o, rays_d = get_rays(test_dirs, td['pose'])
                results = render(model, rays_o, rays_d, test_time=True, exp_step_factor=exp_step_factor)
            if 'rgb' in td:
                psnrs.append(float(psnr_of(F.mse_loss(results['rgb'].float(), td['rgb']))))
                ssims.append(ops.ssim(results['rgb'].float(), td['rgb'], h, w))
            if 'depth' in td:   # mean |D - D^| over the view's pixels with a target
                v = depth_valid(td['depth'])
                if bool(v.any()):
                    depth_maes.append(float((results['depth'].float() - td['depth'])[v].abs().mean()))
            if i == 0:
                from PIL import Image
                img = (results['rgb'].float().clamp(0, 1).reshape(h, w, 3).cpu().numpy() * 255).astype(np.uint8)
                Image.fromarray(img).save(os.path.join(val_dir, 'rgb_000.png'))
                Image.fromarray(depth2img(results['depth'].reshape(h, w).cpu().numpy())).save(
                    os.path.join(val_dir, 'depth_000.png'))
    if psnrs:
        ssim_avg = float(torch.cat(ssims).double().mean())
        print(f"evaluation: psnr_avg={sum(psnrs) / len(psnrs)} | ssim_avg={ssim_avg}"
              + (f" | depth_mae={sum(depth_maes) / len(depth_maes)}" if depth_maes else ""))
    if hparams.extract_mesh:
        save_mesh(model, hparams, os.path.join(val_dir, 'mesh.ply'))

    if hparams.gui:
        from gui import NGPGUI
        hparams.ckpt_path = os.path.join(val_dir, 'model.pth')
        NGPGUI(hparams, model_config, train_dataset.K, train_dataset.img_wh, train_dataset.poses).render()
    return psnrs


if __name__ == '__main__':
    main()
