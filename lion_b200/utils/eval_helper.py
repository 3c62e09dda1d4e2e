"""Scoring a sample file against a reference file (reference utils/eval_helper.py:82-105, 217-340).

Two deliberate differences from the reference's `compute_score`:
  * the reference reads a CD-only switch from the CD_ONLY environment variable when the module is imported; here it is
    the `cd_only` keyword, and a CD-only run returns its results instead of calling exit();
  * there is no comet experiment, visualisation or 'url' entry (`writer` and `exp` are accepted and unused).
"""
import os

import numpy as np
import torch
from loguru import logger

from .data_helper import normalize_point_clouds
from .evaluation_metrics_fast import compute_all_metrics, jsd_between_point_cloud_sets, print_results, write_results

_NUM_TEST = {'animal': 100, 'airplane': 405, 'airplane_ps': 405, 'chair': 662, 'chair_ps': 662, 'car': 352,
             'car_ps': 352, 'all': 1000, 'mug': 22, 'bottle': 43}
_NUM_TEST_LUO = {'airplane': 607, 'chair': 989, 'car': 528}


def get_ref_num(cats, luo_split=False):
    """Number of reference (test) shapes of a category."""
    num_test = _NUM_TEST_LUO if luo_split else _NUM_TEST
    assert cats in num_test, f'not found: {cats} in {num_test}'
    return num_test[cats]


@torch.no_grad()
def compute_score(output_name, ref_name, batch_size_test=256, device_str='cuda', device=None, accelerated_cd=True,
                  writer=None, exp=None, norm_box=False, skip_write=False, cd_only=False, **print_kwargs):
    """MMD / COV / 1-NNA (CD and, unless cd_only, EMD) and JSD of the samples in output_name against the references.

    output_name: a file saved by torch.save holding the samples [S,N,3 or 6] (or a dict whose 'ref' entry does);
    ref_name: a file saved as torch.save({'ref': ref_pcs, 'mean': m_pcs, 'std': s_pcs}).
    The first N_ref = len(ref_pcs) samples are scored.  Samples with more points than the references are subsampled by
    np.random.permutation (seed numpy for a repeatable choice).  With norm_box both sets are bbox-normalised to
    [-0.5, 0.5]; otherwise both are de-normalised with the references' mean and std.  Unless skip_write, the score
    line is appended to results/eval_out.csv.  print_kwargs: dataset, hash, step, epoch of the printed line."""
    logger.info('[compute sample metric] sample: {} and ref: {}', output_name, ref_name)
    ref = torch.load(ref_name, map_location='cpu')
    ref_pcs = ref['ref'][:, :, :3]
    m_pcs, s_pcs = ref['mean'], ref['std']
    gen_pcs = torch.load(output_name, map_location='cpu')
    if isinstance(gen_pcs, dict):
        logger.info('WARNING: the gen_pcs is a dict, with key as {}| usually it is a tensor; '
                    'perhaps this is the train data', gen_pcs.keys())
        gen_pcs = gen_pcs['ref']
    if gen_pcs.shape[1] > ref_pcs.shape[1]:
        keep = np.random.permutation(np.arange(gen_pcs.shape[1]))[:ref_pcs.shape[1]]
        gen_pcs = gen_pcs[:, keep]
    device = torch.device(device_str) if device is None else device
    logger.info('[data shape] ref_pcs: {}, gen_pcs: {}, mean={}, std={}; norm_box={}',
                ref_pcs.shape, gen_pcs.shape, m_pcs.shape, s_pcs.shape, norm_box)
    n_ref = ref_pcs.shape[0]
    m_pcs, s_pcs, ref_pcs, gen_pcs = m_pcs[:n_ref], s_pcs[:n_ref], ref_pcs[:n_ref], gen_pcs[:n_ref]
    if gen_pcs.shape[2] == 6:
        gen_pcs = gen_pcs[:, :, :3]
        ref_pcs = ref_pcs[:, :, :3]
    if norm_box:
        ref_pcs = 0.5 * torch.stack(normalize_point_clouds(ref_pcs), dim=0)
        gen_pcs = 0.5 * torch.stack(normalize_point_clouds(gen_pcs), dim=0)
        print_kwargs['dataset'] = print_kwargs.get('dataset', '') + '-normbox'
    else:
        ref_pcs = ref_pcs * s_pcs + m_pcs
        gen_pcs = gen_pcs * s_pcs + m_pcs
    gen_pcs = gen_pcs.to(device).float()
    ref_pcs = ref_pcs.to(device).float()
    logger.info('print_kwargs: {}', print_kwargs)
    results = compute_all_metrics(gen_pcs, ref_pcs, batch_size_test, accelerated_cd=accelerated_cd,
                                  metric2=None if cd_only else 'EMD', **print_kwargs)
    results['jsd'] = jsd_between_point_cloud_sets(gen_pcs, ref_pcs)
    print_results(results, **print_kwargs)
    if not skip_write:
        os.makedirs('results', exist_ok=True)
        write_results(os.path.join('./results/', 'eval_out.csv'), results, **print_kwargs)
    return results
