"""The reference's SetCriterion / HungarianMatcher (third_party/Mask2Former/mask2former/modeling/criterion.py, matcher.py)
importable on CPU.  oracle.refshim stubs detectron2; the two point_rend helpers the criterion imports are set here to
restatements of detectron2's documented behaviour (detectron2/projects/point_rend/point_features.py):

  point_sample(input, coords)  = F.grid_sample(input, 2 * coords - 1) with coords [N, P, 2] viewed as [N, P, 1, 2]
  get_uncertain_point_coords_with_randomness(logits, f, P, r, beta)
                               = rand(N, int(P * r), 2) candidates; the int(beta * P) with the largest f(sampled
                                 logits) (torch.topk); then rand(N, P - int(beta * P), 2) random points appended."""
import importlib

import torch
import torch.nn.functional as F

from oracle import refshim


def point_sample(input, point_coords, **kwargs):
    add_dim = point_coords.dim() == 3
    if add_dim:
        point_coords = point_coords.unsqueeze(2)
    output = F.grid_sample(input, 2.0 * point_coords - 1.0, **kwargs)
    return output.squeeze(3) if add_dim else output


def get_uncertain_point_coords_with_randomness(coarse_logits, uncertainty_func, num_points, oversample_ratio,
                                               importance_sample_ratio):
    assert oversample_ratio >= 1
    assert 0 <= importance_sample_ratio <= 1
    num_boxes = coarse_logits.shape[0]
    num_sampled = int(num_points * oversample_ratio)
    point_coords = torch.rand(num_boxes, num_sampled, 2, device=coarse_logits.device)
    point_logits = point_sample(coarse_logits, point_coords, align_corners=False)
    point_uncertainties = uncertainty_func(point_logits)
    num_uncertain_points = int(importance_sample_ratio * num_points)
    num_random_points = num_points - num_uncertain_points
    idx = torch.topk(point_uncertainties[:, 0, :], k=num_uncertain_points, dim=1)[1]
    shift = num_sampled * torch.arange(num_boxes, dtype=torch.long, device=coarse_logits.device)
    idx += shift[:, None]
    point_coords = point_coords.view(-1, 2)[idx.view(-1), :].view(num_boxes, num_uncertain_points, 2)
    if num_random_points > 0:
        point_coords = torch.cat(
            [point_coords, torch.rand(num_boxes, num_random_points, 2, device=coarse_logits.device)], dim=1)
    return point_coords


def classes():
    """-> (SetCriterion, HungarianMatcher) of the reference"""
    refshim.install()
    pf = importlib.import_module("detectron2.projects.point_rend.point_features")
    pf.point_sample = point_sample
    pf.get_uncertain_point_coords_with_randomness = get_uncertain_point_coords_with_randomness
    crit = importlib.import_module("mask2former.modeling.criterion")
    match = importlib.import_module("mask2former.modeling.matcher")
    return crit.SetCriterion, match.HungarianMatcher
