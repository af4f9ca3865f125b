"""Command-line flags — same names, defaults and help semantics as the reference's opt.py:4-134 (the
flag table is restated here as data; `--dataset_name synthetic` and the torchrun-related behaviour are
the only additions)."""
import argparse
import math

# (flag, kwargs)
_FLAGS = [
    # dataset parameters
    ('--root_dir', dict(type=str, default='', help='root directory of dataset (unused by the synthetic dataset)')),
    ('--dataset_name', dict(type=str, default='synthetic', choices=['synthetic', 'teacher'],
                            help='synthetic: analytic scene; teacher: views of the reference\'s shipped trained Lego '
                                 'model.  The disk loaders nerf/nsvf/colmap/ngp of the reference are out of scope '
                                 '(SURVEY.md §2.1; no dataset exists offline) and are rejected here')),
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
    ('--tv_sigma_loss_w', dict(type=float, default=0., help='weight of the total-variation loss on the voxel grid\'s '
                                                           'density, 0 to disable (default; svox only)')),
    ('--tv_sh_loss_w', dict(type=float, default=0., help='weight of the total-variation loss on the voxel grid\'s sh '
                                                        'coefficients, 0 to disable (default; svox only)')),
    ('--sparsity_loss_w', dict(type=float, default=0., help='weight of the Cauchy sparsity loss on the voxel grid\'s '
                                                           'densities, 0 to disable (default; svox only)')),
    # training options
    ('--batch_size', dict(type=int, default=8192, help='number of rays in a batch')),
    ('--ray_sampling_strategy', dict(type=str, default='all_images', choices=['all_images', 'same_image'],
                                     help='all_images: uniformly from all pixels of ALL images; '
                                          'same_image: uniformly from all pixels of a SAME image')),
    ('--max_steps', dict(type=int, default=20000, help='number of steps to train')),
    ('--lr', dict(type=float, default=1e-2, help='learning rate')),
    ('--random_bg', dict(action='store_true', default=False, help='train with random bg color (real scene only)')),
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
]

_VOXEL_REG_FLAGS = ('tv_sigma_loss_w', 'tv_sh_loss_w', 'sparsity_loss_w')


def get_opts(prefix_args=None):
    parser = argparse.ArgumentParser()
    for flag, kw in _FLAGS:
        parser.add_argument(flag, **kw)
    hparams = parser.parse_args(prefix_args)
    for flag in _VOXEL_REG_FLAGS:
        w = getattr(hparams, flag)
        if not (math.isfinite(w) and w >= 0):
            parser.error(f"--{flag} must be finite and >= 0, got {w}")
        if w != 0 and hparams.model_name != 'svox':
            parser.error(f"--{flag} regularises the voxel grid: it needs --model_name svox")
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
