"""Oracle of the VLN-CE policy's `waypoint` call with either value of in_train (bevbert_ce/vlnce_baselines/models/
Policy_ViewSelection_BEV.py:166-321), restated with the reference's own torch operations over encoder callables passed
in by the caller, on the CPU or on the CUDA device.  With in_train=True it adds the waypoint augmentation of lines
229-264: every NMS pick is replaced by a cell sampled from its image's regional softmax.

oracle/ce_waypoint_step_ref.py restates the in_train=False branch alone and is the yardstick of the existing tests; the
front of the branch and its candidate loop are restated here again, unchanged, so that the sampling sits where the
reference has it.
"""
import copy
import math

import torch
import torch.nn.functional as F

from .ce_waypoint_step_ref import NUM_ANGLES, NUM_CLASSES, NUM_IMGS, angle_feature_torch


def sample_candidates(probs, noise_rows=None):
    """`torch.distributions.Categorical(probs).sample()` for the (K, 120) regional probabilities of one environment.
    noise_rows (K, 120) replaces the draw: torch.multinomial's single sample is argmax(p / q) over its renormalised
    probabilities p and q = empty_like(p).exponential_(1), so argmax(p / noise_rows) is the sample the reference would
    take had it drawn that noise."""
    probs_c = torch.distributions.Categorical(probs)
    if noise_rows is None:
        return probs_c.sample().detach()
    return torch.argmax(probs_c.probs / noise_rows, dim=-1)


def waypoint_branch(observations, depth_encoder, rgb_encoder, waypoint_predictor, nms, pano_angle_fts, pano_img_idxes,
                    in_train=False, noise=None):
    """BEV.forward(mode='waypoint', in_train=in_train).  depth_encoder(obs) -> (12 B, 128, 4, 4); rgb_encoder(obs) ->
    ((12 B, 512), (12 B, 196, 768)); waypoint_predictor(rgb, depth) -> (B, 120, 12); nms as waypoint_pred/utils.py.
    in_train=True samples with the reference's Categorical(...).sample() when noise is None; otherwise noise[j][:K_j]
    (a (B, 5, 120) tensor, or one (K_j, 120) tensor per environment) is environment j's Exp(1) noise."""
    batch_size = observations['rgb'].shape[0]
    depth_batch = torch.zeros_like(observations['depth']).repeat(NUM_IMGS, 1, 1, 1)
    rgb_batch = torch.zeros_like(observations['rgb']).repeat(NUM_IMGS, 1, 1, 1)
    a_count = 0
    for k, v in observations.items():
        if 'depth' in k:
            for bi in range(v.size(0)):
                ra_count = (NUM_IMGS - a_count) % NUM_IMGS
                depth_batch[ra_count + bi * NUM_IMGS] = v[bi]
                rgb_batch[ra_count + bi * NUM_IMGS] = observations[k.replace('depth', 'rgb')][bi]
            a_count += 1
    obs_view12 = {'depth': depth_batch, 'rgb': rgb_batch}
    depth_embeds = depth_encoder(obs_view12)
    depth_grid_embeds = torch.flatten(F.adaptive_avg_pool2d(depth_batch.permute(0, 3, 1, 2), (14, 14)), 1)
    rgb_embeds, rgb_grid_embeds = rgb_encoder(obs_view12)
    logits = waypoint_predictor(rgb_embeds, depth_embeds)

    rgb_r = rgb_embeds.reshape(batch_size, NUM_IMGS, 512, 1, 1)
    rgb_feats = torch.cat([rgb_r[:, 0:1, :], torch.flip(rgb_r[:, 1:, :], [1])], dim=1)
    dep_r = depth_embeds.reshape(batch_size, NUM_IMGS, 128, 4, 4)
    depth_feats = torch.cat([dep_r[:, 0:1, :], torch.flip(dep_r[:, 1:, :], [1])], dim=1)
    rgb_grid_feats = rgb_grid_embeds.reshape(batch_size, NUM_IMGS, 196, 768)
    depth_grid_feats = depth_grid_embeds.reshape(batch_size, NUM_IMGS, 196, 1)

    x = torch.softmax(logits.reshape(batch_size, NUM_ANGLES * NUM_CLASSES), dim=1)
    x = x.reshape(batch_size, NUM_ANGLES, NUM_CLASSES)
    x = torch.cat((x[:, -1:, :], x, x[:, :1, :]), dim=1)
    out_map = nms(x.unsqueeze(1), max_predictions=5, sigma=(7.0, 5.0)).squeeze(1)[:, 1:-1, :]

    if in_train:
        HEATMAP_OFFSET = 5
        regional = torch.cat((logits[:, -HEATMAP_OFFSET:, :], logits[:, :-HEATMAP_OFFSET, :]), dim=1)
        regional = regional.reshape(batch_size, 12, 10, 12)
        batch_sample_angle_idxes, batch_sample_distance_idxes = [], []
        for j in range(batch_size):
            angle_idxes = out_map[j].nonzero()[:, 0]
            img_idxes = ((angle_idxes.cpu().numpy() + 5) // 10)
            img_idxes[img_idxes == 12] = 0
            way_heats_regional = regional[j][img_idxes].view(img_idxes.size, -1)
            way_heats_probs = F.softmax(way_heats_regional, 1)
            way_heats_act = sample_candidates(way_heats_probs,
                                              None if noise is None else noise[j][:img_idxes.size])
            sample_angle_idxes, sample_distance_idxes = [], []
            for k, way_act in enumerate(way_heats_act):
                if img_idxes[k] != 0:
                    angle_pointer = (img_idxes[k] - 1) * 10 + 5
                else:
                    angle_pointer = 0
                sample_angle_idxes.append(way_act // 12 + angle_pointer)
                sample_distance_idxes.append(way_act % 12)
            batch_sample_angle_idxes.append(sample_angle_idxes)
            batch_sample_distance_idxes.append(sample_distance_idxes)

    rgb_feats = torch.flatten(F.adaptive_avg_pool2d(rgb_feats, (1, 1)), 2)
    depth_feats = torch.flatten(F.adaptive_avg_pool2d(depth_feats, (1, 1)), 2)
    cand_rgb, cand_depth, cand_angle_fts, cand_img_idxes, cand_angles, cand_distances = [], [], [], [], [], []
    for j in range(batch_size):
        if in_train:
            angle_idxes = torch.tensor(batch_sample_angle_idxes[j])
            distance_idxes = torch.tensor(batch_sample_distance_idxes[j])
        else:
            angle_idxes = out_map[j].nonzero()[:, 0]
            distance_idxes = out_map[j].nonzero()[:, 1]
        angle_rad_c = angle_idxes.cpu().float() / 120 * 2 * math.pi
        angle_rad_cc = 2 * math.pi - angle_idxes.float() / 120 * 2 * math.pi
        cand_angle_fts.append(angle_feature_torch(angle_rad_c))
        cand_angles.append(angle_rad_cc.tolist())
        cand_distances.append(((distance_idxes + 1) * 0.25).tolist())
        img_idxes = 12 - (angle_idxes.cpu().numpy() + 5) // 10
        img_idxes[img_idxes == 12] = 0
        cand_img_idxes.append(img_idxes)
        cand_rgb.append(rgb_feats[j, img_idxes, ...])
        cand_depth.append(depth_feats[j, img_idxes, ...])
    return {
        'cand_rgb': cand_rgb, 'cand_depth': cand_depth, 'cand_angle_fts': cand_angle_fts,
        'cand_img_idxes': cand_img_idxes, 'cand_angles': cand_angles, 'cand_distances': cand_distances,
        'pano_rgb': rgb_feats, 'pano_depth': depth_feats, 'pano_rgb_grid': rgb_grid_feats,
        'pano_depth_grid': depth_grid_feats, 'pano_angle_fts': copy.deepcopy(pano_angle_fts),
        'pano_img_idxes': copy.deepcopy(pano_img_idxes),
    }
