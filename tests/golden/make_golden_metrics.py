"""Goldens for the device-side metrics / loss (cspn_b200/csrc/metrics.cu): outputs of the reference's OWN
utils.evaluate_error (/root/reference/cspn_pytorch/utils.py:19-47) and Wighted_L1_Loss (loss.py:16-23, forward and the
gradient autograd gives through it) on seeded inputs, and under metrics/edges/ on inputs with one special value each
(pred 0, -0, negative, +-inf, NaN, subnormal, FLT_MAX; gt at the validity cut and its two neighbours, 0, negative, +inf,
NaN, subnormal; pred == gt), which is what settles how the reference treats them.  tests/test_metrics_gpu.py reads the
files directly under metrics/ with tolerances that a NaN does not survive, hence the subdirectory.
Build container only (needs /root/reference):

    python tests/golden/make_golden_metrics.py
"""
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.join(ROOT, 'tools'))
REF = '/root/reference/cspn_pytorch'
HERE = os.path.dirname(os.path.abspath(__file__))
KEYS = ['MSE', 'RMSE', 'MAE', 'ABS_REL', 'DELTA1.02', 'DELTA1.05', 'DELTA1.10', 'DELTA1.25', 'DELTA1.25^2', 'DELTA1.25^3']


def edge_cases():
    """name -> (gt, pred), 1-D float32: 60 ordinary valid pairs and 4 missing ones, then the special elements.  Each
    poisoning value has a case of its own (one NaN in a sum hides every other), `all_together` holds them all."""
    g = torch.Generator().manual_seed(7)
    base_gt = torch.cat([torch.rand(60, generator=g) * 9.5 + 0.5, torch.zeros(4)])
    base_pred = base_gt * (torch.rand(64, generator=g) * 0.45 + 0.8) + torch.cat([torch.zeros(60), torch.ones(4)])
    cut = np.float32(0.0001)
    inf, nan = float('inf'), float('nan')
    special = {                                  # (gt, pred)
        'pred_zero': (2.0, 0.0), 'pred_negzero': (2.0, -0.0), 'pred_negative': (2.0, -3.0), 'pred_posinf': (2.0, inf),
        'pred_neginf': (2.0, -inf), 'pred_nan': (2.0, nan), 'pred_subnormal': (2.0, 1e-40), 'pred_fltmax': (2.0, 3.4028234663852886e38),
        'gt_cut': (cut, 2.0), 'gt_cut_above': (np.nextafter(cut, np.float32(1)), 2.0),
        'gt_cut_below': (np.nextafter(cut, np.float32(0)), 2.0), 'gt_zero': (0.0, 2.0), 'gt_negative': (-1.0, 2.0),
        'gt_posinf': (inf, 2.0), 'gt_nan': (nan, 2.0), 'gt_subnormal': (1e-40, 2.0),
        'both_posinf': (inf, inf), 'gt_posinf_pred_negative': (inf, -2.0), 'kink': (2.0, 2.0),
    }
    cases = {}
    for name, (a, b) in special.items():
        cases[name] = (torch.cat([base_gt, torch.tensor([a], dtype=torch.float32)]),
                       torch.cat([base_pred, torch.tensor([b], dtype=torch.float32)]))
    cases['all_together'] = (torch.cat([base_gt, torch.tensor([float(a) for a, _ in special.values()], dtype=torch.float32)]),
                             torch.cat([base_pred, torch.tensor([float(b) for _, b in special.values()], dtype=torch.float32)]))
    # every finite special but FLT_MAX at once: nothing poisons or swamps the sums, so their values are checked too
    finite = [k for k, (a, b) in special.items() if np.isfinite(a) and abs(b) < 1e30]
    cases['all_finite'] = (torch.cat([base_gt, torch.tensor([float(special[k][0]) for k in finite], dtype=torch.float32)]),
                           torch.cat([base_pred, torch.tensor([float(special[k][1]) for k in finite], dtype=torch.float32)]))
    return cases


def write_edges(ref_utils, ref_loss):
    os.makedirs(os.path.join(HERE, 'metrics', 'edges'), exist_ok=True)
    for name, (gt, pred) in edge_cases().items():
        err = ref_utils.evaluate_error(gt_depth=gt, pred_depth=pred)
        vals = np.array([float(err[k]) for k in KEYS], dtype=np.float64)
        p = pred.clone().requires_grad_(True)
        loss = ref_loss.Wighted_L1_Loss()(p, gt)
        loss.backward()
        np.savez_compressed(os.path.join(HERE, 'metrics', 'edges', name + '.npz'), gt=gt.numpy(), pred=pred.numpy(),
                            metrics=vals, keys=np.array(KEYS), n_valid=np.int64((gt > 0.0001).sum()),
                            loss=np.float64(loss.item()), grad_pred=p.grad.numpy())
        print('edges/' + name, dict(zip(KEYS, np.round(vals, 5))))


def main():
    from run_reference_eval import _stub_modules
    _stub_modules()                                  # utils.py imports matplotlib / skimage, absent here
    sys.path[:0] = [REF, os.path.join(REF, 'models')]
    import loss as ref_loss
    import utils as ref_utils
    cases = {
        'nyu_like': (3, (2, 1, 228, 304), 0.0, 1.0),          # dense ground truth
        'kitti_like': (4, (2, 1, 64, 256), 0.7, 1.0),         # 70 % of the ground truth missing (== 0)
        'close_prediction': (5, (1, 1, 40, 60), 0.2, 0.02),   # errors around the delta thresholds
        'nothing_valid': (6, (1, 1, 8, 8), 1.0, 1.0),
    }
    for name, (seed, shape, p_missing, noise) in cases.items():
        g = torch.Generator().manual_seed(seed)
        gt = torch.rand(shape, generator=g) * 10
        gt = gt * (torch.rand(shape, generator=g) >= p_missing).float()
        pred = (gt + noise * torch.randn(shape, generator=g)).clamp_min(0.05) if noise < 1 else torch.rand(shape, generator=g) * 10
        err = ref_utils.evaluate_error(gt_depth=gt, pred_depth=pred)
        vals = np.array([float(err[k]) for k in KEYS], dtype=np.float64)
        rec = dict(gt=gt.numpy(), pred=pred.numpy(), metrics=vals, keys=np.array(KEYS))
        if (gt > 0.0001).any():
            p = pred.clone().requires_grad_(True)
            loss = ref_loss.Wighted_L1_Loss()(p, gt)
            loss.backward()
            rec.update(loss=np.float64(loss.item()), grad_pred=p.grad.numpy())
        np.savez_compressed(os.path.join(HERE, 'metrics', name + '.npz'), **rec)
        print(name, dict(zip(KEYS, np.round(vals, 5))))
    write_edges(ref_utils, ref_loss)


if __name__ == '__main__':
    main()
