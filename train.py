"""Training entry point — same CLI and loop structure as the reference's train.py (main() :35-322):
seeds (:39-42), model_config (:86-117), mark_invisible_cells (:129), loss scale 2**16 | 2**19 (:137-141),
Adam(lr, eps=1e-15) + cosine annealing to lr/30 (:143-163), density-grid update every 16 steps with a
256-step warm-up (:57-58,178-182), log line every 1000 steps (:203-219), results/model.pth (:232-235),
test-split PSNR (:237-304).  The step body runs on the sm_90a kernels through NGPTrainer (fused Adam,
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
from modules.distortion import distortion_loss
from modules.networks import MODEL_DICT
from modules.rendering import MAX_SAMPLES, render
from modules.utils import depth2img, save_deployment_model
from opt import get_opts
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
    extra = {'scene': 'analytic'} if hparams.dataset_name == 'synthetic' else {}
    train_dataset = dataset(root_dir=hparams.root_dir, split=hparams.split, downsample=hparams.downsample,
                            seed=seed, **extra).to(device)
    train_dataset.batch_size = hparams.batch_size
    train_dataset.ray_sampling_strategy = hparams.ray_sampling_strategy
    if hparams.random_bg:
        raise SystemExit("--random_bg applies to real scenes with an alpha channel (datasets/colmap.py of the "
                         "reference), which are out of scope here (SURVEY.md §2.1)")
    train_dataset._seed = seed + rank  # different rays per rank
    test_dataset = dataset(root_dir=hparams.root_dir, split='test', downsample=hparams.downsample,
                           n_images=4, **extra).to(device)

    model_config = build_model_config(hparams)
    model = MODEL_DICT[hparams.model_name](**model_config).to(device)
    if hparams.ckpt_path:
        model.load_state_dict(torch.load(hparams.ckpt_path, map_location=device))
        print("Load checkpoint from %s" % hparams.ckpt_path)
    model.mark_invisible_cells(train_dataset.K, train_dataset.poses, train_dataset.img_wh)

    torch.manual_seed(seed + rank)  # data / marching noise differ per rank from here on
    voxel_reg = None
    if hparams.model_name == 'svox':   # total variation / sparsity weights; all 0 (the default) enqueue nothing
        voxel_reg = (hparams.tv_sigma_loss_w, hparams.tv_sh_loss_w, hparams.sparsity_loss_w)
    trainer = NGPTrainer(model, lr=hparams.lr, max_steps=hparams.max_steps, voxel_reg=voxel_reg)

    fast = None
    if hparams.graph_step:
        if not model._fusable(next(model.parameters())):
            raise ValueError("--graph_step needs the stock NGP architecture")
        if getattr(model, 'pos_encoder_type', 'hash') != 'hash':
            raise ValueError("--graph_step runs the hash encoder only; train a tri-plane model without it")
        from taichi_nerfs_b200.fast_step import StaticTrainStep
        fast = StaticTrainStep(trainer, hparams.batch_size, exp_step_factor=exp_step_factor,
                               distortion_loss_w=hparams.distortion_loss_w)

    tic = time.time()
    for step in range(hparams.max_steps + 1):
        model.train()
        data = train_dataset[step % len(train_dataset)]
        with torch.autocast(device_type='cuda', dtype=torch.float16):
            if step % update_interval == 0:
                model.update_density_grid(0.01 * MAX_SAMPLES / 3 ** 0.5, warmup=step < warmup_steps)
        rays_o, rays_d = get_rays(data['direction'], data['pose'])
        extra_loss = None
        if hparams.distortion_loss_w > 0:
            extra_loss = lambda res: hparams.distortion_loss_w * distortion_loss(res).mean()  # noqa: E731
        if fast is not None:   # one graph replay, nothing synchronises the host
            loss = fast.step(rays_o, rays_d, data['rgb'])
            results = {'rgb': fast.rgb, 'rm_samples': fast.counter[0].clamp(max=fast.cap), 'vr_samples':
                       fast.counter[0].clamp(max=fast.cap), 'dropped_rays': fast.counter[1]}
        else:
            loss, results = trainer.step(rays_o, rays_d, data['rgb'], exp_step_factor, extra_loss=extra_loss)

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

    # test loop (train.py:237-304): PSNR per held-out view; first view saved as PNG
    model.eval()
    w, h = test_dataset.img_wh
    psnrs = []
    with torch.no_grad():
        for i in range(len(test_dataset)):
            td = test_dataset[i]
            with torch.autocast(device_type='cuda', dtype=torch.float16):
                rays_o, rays_d = get_rays(test_dataset.directions, td['pose'])
                results = render(model, rays_o, rays_d, test_time=True, exp_step_factor=exp_step_factor)
            if 'rgb' in td:
                psnrs.append(float(psnr_of(F.mse_loss(results['rgb'].float(), td['rgb']))))
            if i == 0:
                from PIL import Image
                img = (results['rgb'].float().clamp(0, 1).reshape(h, w, 3).cpu().numpy() * 255).astype(np.uint8)
                Image.fromarray(img).save(os.path.join(val_dir, 'rgb_000.png'))
                Image.fromarray(depth2img(results['depth'].reshape(h, w).cpu().numpy())).save(
                    os.path.join(val_dir, 'depth_000.png'))
    if psnrs:
        print(f"evaluation: psnr_avg={sum(psnrs) / len(psnrs)}")

    if hparams.gui:
        from gui import NGPGUI
        hparams.ckpt_path = os.path.join(val_dir, 'model.pth')
        NGPGUI(hparams, model_config, train_dataset.K, train_dataset.img_wh, train_dataset.poses).render()
    return psnrs


if __name__ == '__main__':
    main()
