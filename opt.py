"""Command-line flags — same names, defaults and help semantics as the reference's opt.py:4-134 (the
flag table is restated here as data; `--dataset_name synthetic | teacher` and the torchrun-related behaviour
are the additions)."""
import argparse
import math
import os

# (flag, kwargs)
_FLAGS = [
    # dataset parameters
    ('--root_dir', dict(type=str, default='', help='root directory of dataset (needed by nerf, nsvf, colmap and ngp; '
                                                  'unused by synthetic and teacher)')),
    ('--dataset_name', dict(type=str, default='synthetic', choices=['synthetic', 'teacher', 'nerf', 'nsvf', 'colmap',
                                                                     'ngp'],
                            help='synthetic: analytic scene; teacher: views of the reference\'s shipped trained Lego '
                                 'model; nerf (Blender transforms_*.json), nsvf, colmap (sparse/0/*.bin), ngp '
                                 '(transforms.json): the reference\'s disk loaders, reading --root_dir')),
    ('--split', dict(type=str, default='train', choices=['train', 'trainval', 'trainvaltest'],
                     help='use which split to train')),
    ('--downsample', dict(type=float, default=1.0, help='downsample factor (<=1.0) for the images')),
    # model parameters
    ('--model_name', dict(type=str, default='ngp', choices=['ngp', 'svox'],
                          help='which model to train/test: ngp (hash or tri-plane encoder + MLPs) or svox (voxel grid '
                               'of spherical-harmonics coefficients and densities; not with --encoder_type triplane, '
                               '--graph_step or --deployment)')),
    ('--scale', dict(type=float, default=0.5, help='scene scale (whole scene must lie in [-scale, scale]^3')),
    ('--half_opt', dict(action='store_true', default=False, help='whether to use half optimization')),
    ('--encoder_type', dict(type=str, default='hash', choices=['hash', 'triplane'],
                        help='which encoder to use: the multiresolution hash grid or the tri-plane encoder (fp32 '
                             'planes; not with --half_opt or --deployment; --graph_step is not wired to it yet, '
                             'StaticTrainStep runs it)')),
    ('--sh_degree', dict(type=int, default=2, help='degree of spherical harmonics: 0, 1 or 2 (svox only)')),
    ('--grid_size', dict(type=int, default=256, help='nodes of the voxel grid in each dimension (svox only; the '
                                                     'occupancy grid stays 128^3)')),
    ('--grid_radius', dict(type=float, default=0.0125, help='spacing of the voxel grid nodes (svox only)')),
    ('--origin_sh', dict(type=float, default=0., help='initial value of the sh coefficients in the voxel grid '
                                                      '(svox only)')),
    ('--origin_sigma', dict(type=float, default=0.1, help='initial value of the density in the voxel grid '
                                                          '(svox only)')),
    # loss parameters
    ('--distortion_loss_w', dict(type=float, default=0, help='weight of distortion loss, 0 to disable (default)')),
    ('--depth_loss_w', dict(type=float, default=0.,
                            help='weight of the depth loss w mean(v (D - D^)^2) against per-ray target z-depth, 0 to '
                                 'disable (default); needs a dataset with depth: ngp (depth_path), synthetic, teacher')),
    ('--tv_sigma_loss_w', dict(type=float, default=0., help='weight of the total-variation loss on the voxel grid\'s '
                                                           'density, 0 to disable (default; svox only)')),
    ('--tv_sh_loss_w', dict(type=float, default=0., help='weight of the total-variation loss on the voxel grid\'s sh '
                                                        'coefficients, 0 to disable (default; svox only)')),
    ('--sparsity_loss_w', dict(type=float, default=0., help='weight of the Cauchy sparsity loss on the voxel grid\'s '
                                                           'densities, 0 to disable (default; svox only)')),
    # training options
    ('--batch_size', dict(type=int, default=8192, help='number of rays in a batch')),
    ('--ray_sampling_strategy', dict(type=str, default='all_images', choices=['all_images', 'same_image', 'error_map'],
                                     help='all_images: uniformly from all pixels of ALL images; '
                                          'same_image: uniformly from all pixels of a SAME image; '
                                          'error_map: from all pixels of all images in proportion to their tile\'s '
                                          'recent error, each ray\'s loss weighted to keep the objective unbiased '
                                          '(DESIGN.md §6j; one GPU)')),
    ('--error_map_res', dict(type=int, default=64,
                             help='tiles per image side of the error map (clamped to the image size), '
                                  'with --ray_sampling_strategy error_map')),
    ('--max_steps', dict(type=int, default=20000, help='number of steps to train')),
    ('--lr', dict(type=float, default=1e-2, help='learning rate')),
    ('--random_bg', dict(action='store_true', default=False, help='train with random bg color (real scene only)')),
    ('--extrinsics_lr', dict(type=float, default=0.,
                             help='learning rate of the per-image camera pose corrections (rotation and translation, '
                                  'DESIGN.md §6i), 0 to disable (default); hash encoder only, one GPU')),
    ('--exposure_lr', dict(type=float, default=0.,
                           help='learning rate of the per-image exposures (a log2 gain per colour channel, DESIGN.md '
                                '§6k), 0 to disable (default); every model kind, one GPU')),
    ('--lens_distortion', dict(action='store_true', default=False,
                               help='keep the lens distortion of the COLMAP camera or transforms.json (k1 k2 p1 p2) '
                                    'and unproject every pixel through it (DESIGN.md §6l); --dataset_name colmap | ngp')),
    ('--intrinsics_lr', dict(type=float, default=0.,
                             help='learning rate of the camera intrinsics corrections (log focal scale and principal '
                                  'point, DESIGN.md §6l), 0 to disable (default); hash encoder only, one GPU')),
    # misc
    ('--exp_name', dict(type=str, default='exp', help='experiment name')),
    ('--gpu', dict(type=int, default=0, help='set cuda device (ignored under torchrun: LOCAL_RANK wins)')),
    ('--ckpt_path', dict(type=str, default=None, help='pretrained checkpoint to load')),
    ('--gui', dict(action='store_true', default=False, help='render an orbit with the GUI camera after training')),
    ('--graph_step', dict(action='store_true', default=False,
                          help='run the training step as one CUDA-graph replay (StaticTrainStep; stock NGP '
                               'architecture, --distortion_loss_w included; this switch takes the hash encoder only); '
                               'same update as '
                               'the default module path')),
    ('--deployment', dict(action='store_true', default=False)),
    ('--deployment_model_path', dict(type=str, default='./')),
    # mesh export (DESIGN.md §6g)
    ('--extract_mesh', dict(action='store_true', default=False,
                            help='after evaluation, write results/mesh.ply: marching cubes over the density lattice')),
    ('--mesh_res', dict(type=int, default=512, help='lattice nodes per axis of the mesh export, in [2, 1024]')),
    ('--mesh_threshold', dict(type=float, default=10.0, help='density above which a lattice node is inside the mesh')),
    ('--mesh_bound', dict(type=float, default=0.0, help='half-width of the meshed cube, in (0, scale]; 0 means scale')),
]

_VOXEL_REG_FLAGS = ('tv_sigma_loss_w', 'tv_sh_loss_w', 'sparsity_loss_w')
DISK_DATASETS = ('nerf', 'nsvf', 'colmap', 'ngp')


def get_opts(prefix_args=None):
    parser = argparse.ArgumentParser()
    for flag, kw in _FLAGS:
        parser.add_argument(flag, **kw)
    hparams = parser.parse_args(prefix_args)
    if not 2 <= hparams.mesh_res <= 1024:
        parser.error(f"--mesh_res must be in [2, 1024], got {hparams.mesh_res}")
    if not math.isfinite(hparams.mesh_threshold):
        parser.error(f"--mesh_threshold must be finite, got {hparams.mesh_threshold}")
    if not (hparams.mesh_bound == 0 or (math.isfinite(hparams.mesh_bound) and 0 < hparams.mesh_bound <= hparams.scale)):
        parser.error(f"--mesh_bound must be 0 (meaning --scale) or in (0, {hparams.scale}], got {hparams.mesh_bound}")
    if hparams.dataset_name in DISK_DATASETS and not hparams.root_dir:
        parser.error(f"--dataset_name {hparams.dataset_name} reads a dataset from disk: it needs --root_dir")
    for flag in _VOXEL_REG_FLAGS:
        w = getattr(hparams, flag)
        if not (math.isfinite(w) and w >= 0):
            parser.error(f"--{flag} must be finite and >= 0, got {w}")
        if w != 0 and hparams.model_name != 'svox':
            parser.error(f"--{flag} regularises the voxel grid: it needs --model_name svox")
    if not (math.isfinite(hparams.depth_loss_w) and hparams.depth_loss_w >= 0):
        parser.error(f"--depth_loss_w must be finite and >= 0, got {hparams.depth_loss_w}")
    if hparams.depth_loss_w > 0 and hparams.dataset_name in ('nerf', 'nsvf', 'colmap'):
        parser.error(f"--depth_loss_w: the {hparams.dataset_name} loader reads no depth (the ngp loader reads "
                     f"transforms.json's depth_path)")
    if not 1 <= hparams.error_map_res <= 4096:
        parser.error(f"--error_map_res must be in [1, 4096], got {hparams.error_map_res}")
    if hparams.ray_sampling_strategy == 'error_map' and int(os.environ.get("WORLD_SIZE", "1")) > 1:
        parser.error("--ray_sampling_strategy error_map trains on one GPU: the error map is not shared between ranks")
    if not (math.isfinite(hparams.extrinsics_lr) and hparams.extrinsics_lr >= 0):
        parser.error(f"--extrinsics_lr must be finite and >= 0, got {hparams.extrinsics_lr}")
    if hparams.extrinsics_lr > 0:
        if not (math.isfinite(hparams.lr) and hparams.lr > 0):
            parser.error(f"--extrinsics_lr is set relative to the model's learning rate: it needs a finite --lr > 0, got "
                         f"{hparams.lr}")
        if hparams.model_name == 'svox':
            parser.error("--extrinsics_lr does not combine with --model_name svox: the voxel grid gives no gradient "
                         "wrt the sample positions")
        if hparams.encoder_type == 'triplane':
            parser.error("--extrinsics_lr does not combine with --encoder_type triplane: the tri-plane encoder gives no "
                         "gradient wrt the sample positions")
    if hparams.lens_distortion and hparams.dataset_name not in ('colmap', 'ngp'):
        parser.error(f"--lens_distortion reads the distortion terms of a COLMAP camera or transforms.json: it needs "
                     f"--dataset_name colmap | ngp, got {hparams.dataset_name}")
    if not (math.isfinite(hparams.intrinsics_lr) and hparams.intrinsics_lr >= 0):
        parser.error(f"--intrinsics_lr must be finite and >= 0, got {hparams.intrinsics_lr}")
    if hparams.intrinsics_lr > 0:
        if not (math.isfinite(hparams.lr) and hparams.lr > 0):
            parser.error(f"--intrinsics_lr is set relative to the model's learning rate: it needs a finite --lr > 0, got "
                         f"{hparams.lr}")
        if hparams.model_name == 'svox':
            parser.error("--intrinsics_lr does not combine with --model_name svox: the voxel grid gives no gradient "
                         "wrt the sample positions")
        if hparams.encoder_type == 'triplane':
            parser.error("--intrinsics_lr does not combine with --encoder_type triplane: the tri-plane encoder gives no "
                         "gradient wrt the sample positions")
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            parser.error("--intrinsics_lr trains on one GPU: the intrinsics gradient is not exchanged between ranks")
    if not (math.isfinite(hparams.exposure_lr) and hparams.exposure_lr >= 0):
        parser.error(f"--exposure_lr must be finite and >= 0, got {hparams.exposure_lr}")
    if hparams.exposure_lr > 0:
        if not (math.isfinite(hparams.lr) and hparams.lr > 0):
            parser.error(f"--exposure_lr is set relative to the model's learning rate: it needs a finite --lr > 0, got "
                         f"{hparams.lr}")
        if int(os.environ.get("WORLD_SIZE", "1")) > 1:
            parser.error("--exposure_lr trains on one GPU: the exposure gradient is not exchanged between ranks")
    if hparams.model_name == 'svox':
        for flag, bad, why in (
                ('encoder_type', hparams.encoder_type == 'triplane',
                 'the voxel grid has no position encoder (--encoder_type applies to ngp)'),
                ('graph_step', hparams.graph_step,
                 'the graph-captured step runs the NGP encoder + MLP kernels; train the voxel grid without it'),
                ('deployment', hparams.deployment, 'the deployment export (mobile demo format) is hash-only')):
            if bad:
                parser.error(f"--model_name svox does not combine with --{flag}"
                             f"{' triplane' if flag == 'encoder_type' else ''}: {why}")
    if hparams.encoder_type == 'triplane':
        for flag, why in (('half_opt', 'the tri-plane table is fp32 (an fp16 plane table is not supported)'),
                          ('graph_step', 'this switch is not wired to the tri-plane encoder yet (the graph-captured step '
                                         'itself runs it: taichi_nerfs_b200.fast_step.StaticTrainStep)'),
                          ('deployment', 'the deployment export (mobile demo format) is hash-only')):
            if getattr(hparams, flag):
                parser.error(f"--encoder_type triplane does not combine with --{flag}: {why}")
    return hparams
