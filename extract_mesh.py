"""Mesh export from a checkpoint (DESIGN.md §6g): the model flags of train.py plus --ckpt_path, and the --mesh_*
flags; writes results/mesh.ply, the same bytes train.py --extract_mesh writes for the same model.

    python extract_mesh.py --ckpt_path results/model.pth --mesh_res 512 --mesh_threshold 10
"""
import os

import torch

from modules.networks import MODEL_DICT
from opt import get_opts
from train import build_model_config, save_mesh


def main(prefix_args=None):
    hparams = get_opts(prefix_args)
    if not hparams.ckpt_path:
        raise SystemExit("extract_mesh.py needs --ckpt_path (a state_dict written by train.py)")
    if not torch.cuda.is_available():
        raise RuntimeError("extract_mesh.py needs a CUDA device: the mesh kernels have no CPU fallback")
    device = torch.device("cuda", max(hparams.gpu, 0))
    torch.cuda.set_device(device)
    model = MODEL_DICT[hparams.model_name](**build_model_config(hparams)).to(device)
    model.load_state_dict(torch.load(hparams.ckpt_path, map_location=device))   # occupancy buffers included
    model.eval()
    os.makedirs('results', exist_ok=True)
    path = os.path.join('results', 'mesh.ply')
    save_mesh(model, hparams, path)
    return path


if __name__ == '__main__':
    main()
