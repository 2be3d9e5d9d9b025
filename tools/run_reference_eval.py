"""Runs the REFERENCE's own evaluation driver -- /root/reference/cspn_pytorch/eval.py, unmodified, top to bottom including its
`val()` loop (:130-168) -- on torch 2.x / numpy 2.x without the NYU dataset:

    python tools/run_reference_eval.py [--reference /root/reference/cspn_pytorch] [--cspn dropin|reference] [--samples 2]

What is supplied around it (nothing inside the reference tree is touched):
  * a stub `eval_nyu_dataset_loader` module whose NyuDepthDataset yields seeded random 228x304 RGB-D samples in the loader's
    format ({'rgbd', 'depth', 'raw_rgb'}, nyu_dataset_loader.py:49-133) -- the real one needs h5py, skimage and 32 GB of data;
  * empty stand-ins for modules the box lacks (matplotlib, skimage, h5py) and the numpy-2 names the reference still uses
    (`np.int`, nyu_dataset_loader.py:81; `np.Inf`, lr_scheduler.py:69);
  * a checkpoint directory with a `best_model.pth` of seeded random weights in the reference's own format (DataParallel
    `module.` prefix plus the stray `post_process_layer.sum_conv.weight` every reference checkpoint carries);
  * `--cspn dropin`: `dropin/` goes on sys.path BEFORE the reference's ./models (eval.py:52 appends it), so
    torch_resnet_cspn_nyu.py:12 (`import cspn as post_process`) resolves to the CUDA module: needs a GPU.
    `--cspn reference`: the reference's own cspn.py (CPU works: `.cuda()` becomes the identity where CUDA is absent).
Returns / prints the model outputs eval.py computed, so the two choices can be compared: same weights, same samples.
"""
import argparse
import os
import runpy
import sys
import tempfile
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _stub_modules():
    for name in ('matplotlib', 'matplotlib.pyplot', 'skimage', 'skimage.io', 'skimage.transform', 'h5py'):
        if name not in sys.modules:
            try:
                __import__(name)
            except Exception:
                sys.modules[name] = types.ModuleType(name)
                if '.' in name:
                    setattr(sys.modules[name.split('.')[0]], name.split('.')[1], sys.modules[name])
    if not hasattr(np, 'int'):
        np.int = int          # nyu_dataset_loader.py:81
    if not hasattr(np, 'Inf'):
        np.Inf = np.inf       # lr_scheduler.py:69


def _stub_loader(n_samples, seed):
    mod = types.ModuleType('eval_nyu_dataset_loader')

    class NyuDepthDataset(torch.utils.data.Dataset):
        """Same sample format as the reference loader: 'rgbd' 4x228x304 (RGB + sparse depth), 'depth' 1x228x304."""

        def __init__(self, csv_file=None, root_dir=None, split='val', n_sample=200, input_format='hdf5'):
            self.n_sample = n_sample

        def __len__(self):
            return n_samples

        def __getitem__(self, idx):
            g = torch.Generator().manual_seed(seed + idx)
            rgb = torch.rand(3, 228, 304, generator=g)
            depth = torch.rand(1, 228, 304, generator=g) * 10
            keep = (torch.rand(1, 228, 304, generator=g) < self.n_sample / (228.0 * 304.0)).float()   # nyu_dataset_loader.py:135-144
            return {'rgbd': torch.cat([rgb, depth * keep], 0), 'depth': depth, 'raw_rgb': rgb.clone()}

    mod.NyuDepthDataset = NyuDepthDataset
    return mod


def run_eval(reference, cspn='dropin', samples=2, seed=7, quiet=True):
    """Executes eval.py; returns the list of output tensors (one per sample, CPU) its val() loop produced."""
    models = os.path.join(reference, 'models')
    assert os.path.isfile(os.path.join(reference, 'eval.py')), f'{reference}/eval.py not found'
    _stub_modules()
    saved = dict(path=list(sys.path), argv=list(sys.argv), cwd=os.getcwd(), cuda=torch.Tensor.cuda, mcuda=torch.nn.Module.cuda)
    touched = ('cspn', 'torch_resnet_cspn_nyu', 'update_model', 'utils', 'loss', 'data_transform', 'eval_nyu_dataset_loader')
    for name in touched:
        sys.modules.pop(name, None)
    outputs = []
    work = tempfile.mkdtemp(prefix='cspn_eval_')
    try:
        if not torch.cuda.is_available():
            torch.Tensor.cuda = lambda self, *a, **k: self          # cspn.py:50 and Unpool's ctor call .cuda() unconditionally
            torch.nn.Module.cuda = lambda self, *a, **k: self       # eval.py:126: criterion = Wighted_L1_Loss().cuda()
        sys.path[:0] = ([os.path.join(ROOT, 'dropin'), ROOT] if cspn == 'dropin' else []) + [reference]
        sys.path.append(models)                                        # what eval.py:52 does itself, relative to its cwd
        sys.modules['eval_nyu_dataset_loader'] = _stub_loader(samples, seed)
        import utils as ref_utils                                      # the reference's utils.py (reference root is on sys.path)
        ref_utils.save_eval_img = lambda data_set, model_dir, index, rgbd, rgb, gt, pred: outputs.append(pred.clone())
        # a checkpoint in the reference's own format, from a seeded random model built by the reference's own code
        import torch_resnet_cspn_nyu as ref_model
        torch.manual_seed(seed)
        net = ref_model.resnet50(cspn_config={'step': 24, 'norm_type': '8sum'})
        sd = {'module.' + k: v for k, v in net.state_dict().items()}
        sd['module.post_process_layer.sum_conv.weight'] = torch.ones(1, 8, 1, 1, 1)
        torch.save(sd, os.path.join(work, 'best_model.pth'))
        del net, sd
        os.chdir(work)
        os.makedirs('models', exist_ok=True)
        sys.argv = ['eval.py', '--model', 'cspn_unet', '--data_set', 'nyudepth', '--best_model_dir', work,
                    '--batch_size_eval', '1', '--n_sample', '500', '--cspn_step', '24', '--cspn_norm_type', '8sum']
        if quiet:
            import contextlib
            import io
            with contextlib.redirect_stdout(io.StringIO()):
                runpy.run_path(os.path.join(reference, 'eval.py'), run_name='__main__')
        else:
            runpy.run_path(os.path.join(reference, 'eval.py'), run_name='__main__')
        which = sys.modules['torch_resnet_cspn_nyu'].post_process.__file__
    finally:
        os.chdir(saved['cwd'])
        sys.path[:] = saved['path']
        sys.argv[:] = saved['argv']
        torch.Tensor.cuda = saved['cuda']
        torch.nn.Module.cuda = saved['mcuda']
        for name in touched:
            sys.modules.pop(name, None)
    return outputs, which


if __name__ == '__main__':
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument('--reference', default='/root/reference/cspn_pytorch')
    ap.add_argument('--cspn', default='dropin', choices=['dropin', 'reference'])
    ap.add_argument('--samples', type=int, default=2)
    a = ap.parse_args()
    outs, which = run_eval(a.reference, a.cspn, a.samples, quiet=False)
    print(f'eval.py ran to completion: {len(outs)} samples through {which}; output checksums',
          [round(float(o.double().sum()), 6) for o in outs])
