"""Dataset registry.  The reference's four disk loaders (nerf, nsvf, ngp, colmap; DESIGN.md §6f) read the
formats the reference's training scripts pass with ``--root_dir``; the synthetic Lego-shape set drives the
benchmark and the teacher set (views of the reference's shipped trained Lego model) the PSNR protocol."""
from .colmap import ColmapDataset
from .nerf import NeRFDataset
from .ngp import NGPDataset
from .nsvf import NSVFDataset
from .synthetic import SyntheticLego
from .teacher import TeacherLego

dataset_dict = {'synthetic': SyntheticLego, 'teacher': TeacherLego, 'nerf': NeRFDataset, 'nsvf': NSVFDataset,
                'colmap': ColmapDataset, 'ngp': NGPDataset}
