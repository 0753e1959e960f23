"""The agents' per-step BEV input built by one kernel straight from the navigation graph's node clouds.

`nav_bev_variable(agent, obs, gmaps)` returns the dict of the reference agents' `_nav_bev_variable`
(map_nav_src/r2r/agent.py:293-337, identical in reverie/agent_obj.py, which the SOON agent inherits):
`bev_fts, bev_pos_fts, bev_masks, bev_nav_masks, bev_cand_idxs, bev_cand_vpids`.  Only the point-cloud half changes:
instead of `torch.cat`-ing the clouds of the current node and its neighbours (`GraphMap.gather_node_pc`), padding them
into a batch (`pad_sequence`), transforming them to the ego frame (`splat`) and pooling them (`project_bev`), one
`bb_bev_splat_nodes` launch reads every node cloud where `GraphMap.node_pc` keeps it.  Everything else goes through the
agent's own methods (`_map_cand_to_bev`, `GraphMap.get_pos_fts`, `graph.path`, `bev_pos`, `args.pc_order`).

Install on an agent once it is built:

    agent._nav_bev_variable = types.MethodType(nav_bev_variable, agent)
"""
import numpy as np
import torch

from . import bev_nodes

Y_CLIP = 0.5    # height clip of the agents' project_bev (map_nav_src/models/bev_utils.py:398)


def gathered_nodes(gmap, vp, order):
    """The viewpoints whose clouds `GraphMap.gather_node_pc(vp, order)` concatenates, in its order: the node alone at
    order 0, otherwise every node with a cloud, in insertion order of `node_pc`, at most `order` graph hops from vp."""
    if order == 0:
        return [vp]
    return [c for c in gmap.node_pc if len(gmap.graph.path(vp, c)) <= order]


def ego_frames(obs):
    """World -> ego transform of each sample, float32: S (B,3) = (x, z, -y) of the agent's position and T (B,4,4) a
    rotation about the vertical axis by the heading, built in float64 and rounded to float32 like the agents'
    matrices (agent.py:150-159)."""
    h = np.array([o["heading"] for o in obs], dtype=np.float64)
    c, s = np.cos(h), np.sin(h)
    S = np.array([[o["position"][0], o["position"][2], -o["position"][1]] for o in obs], dtype=np.float64)
    T = np.zeros((len(obs), 4, 4), dtype=np.float64)
    T[:, 0, 0], T[:, 0, 2] = c, s
    T[:, 1, 1] = 1.0
    T[:, 2, 0], T[:, 2, 2] = -s, c
    T[:, 3, 3] = 1.0
    return S.astype(np.float32), T.astype(np.float32)


def nav_bev_variable(agent, obs, gmaps):
    """Drop-in for the agents' `_nav_bev_variable(obs, gmaps)`; see the module docstring."""
    B, D = len(obs), agent.bev_dim
    clouds = [[gmap.node_pc[c] for c in gathered_nodes(gmap, ob["viewpoint"], agent.args.pc_order)]
              for ob, gmap in zip(obs, gmaps)]
    dev = next((n[0].device for nodes in clouds for n in nodes), agent.bev_pos.device)

    nav_masks = np.zeros((B, D * D), dtype=bool)
    cand_idxs, cand_vpids, gpos = [], [], []
    for i, (ob, gmap) in enumerate(zip(obs, gmaps)):
        cand_vpids.append([None] + [c["viewpointId"] for c in ob["candidate"]])     # None: the stop action
        pos = agent._map_cand_to_bev(ob)
        idx = np.insert(pos[:, 1] * D + pos[:, 0], 0, (D * D - 1) // 2)            # stop sits on the centre cell
        nav_masks[i, idx] = True
        cand_idxs.append(idx)
        gpos.append(gmap.get_pos_fts(ob["viewpoint"], [gmap.start_vp], ob["heading"], ob["elevation"]))

    S, T = ego_frames(obs)
    frames = torch.from_numpy(np.concatenate([S.ravel(), T.ravel()])).to(dev)     # one upload for both
    bev_fts, _ = bev_nodes.bev_splat_nodes(clouds, frames[:3 * B].view(B, 3), frames[3 * B:].view(B, 4, 4), D,
                                           agent.bev_res, Y_CLIP)

    L = max(len(c) for c in cand_idxs)
    bev_cand_idxs = torch.zeros(B, L, dtype=torch.from_numpy(cand_idxs[0]).dtype)
    for i, c in enumerate(cand_idxs):
        bev_cand_idxs[i, :len(c)] = torch.from_numpy(c)
    gpos = torch.from_numpy(np.stack(gpos, 0)).to(dev)
    return {
        "bev_fts": bev_fts,
        "bev_pos_fts": torch.cat([gpos.expand(-1, D * D, -1), agent.bev_pos.reshape(B, -1, 3)], -1),
        "bev_masks": torch.ones(B, D * D, dtype=torch.bool, device=dev),
        "bev_nav_masks": torch.from_numpy(nav_masks).to(dev),
        "bev_cand_idxs": bev_cand_idxs,
        "bev_cand_vpids": cand_vpids,
    }
