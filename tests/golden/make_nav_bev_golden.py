"""Generates tests/golden/nav_bev.pt, the pin of tests/test_nav_bev_cpu.py, by running the UNMODIFIED reference's
map_nav_src GraphMap and PointCloud.project_bev (located by oracle/ref_shim.py, env BEVBERT_REFERENCE) on the synthetic
episode of tests/nav_bev_cases.py:

    PYTHONDONTWRITEBYTECODE=1 BEVBERT_REFERENCE=<reference checkout> python tests/golden/make_nav_bev_golden.py

The episode is regenerated bit-identically from its seed by the test, so only reference OUTPUTS are stored."""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from oracle import ref_shim  # noqa: E402
from oracle.bevbert_ref import cell_index  # noqa: E402


def sample_rows(x, n=16, seed=0):
    """Fixed, seeded sample of n rows of x flattened to 2-D, plus float64 sums of the whole tensor (the layout of
    make_golden.py's pins)."""
    x2 = x.reshape(-1, x.shape[-1]).detach()
    idx = torch.randperm(x2.shape[0], generator=torch.Generator().manual_seed(seed))[:n].sort().values
    return {"idx": idx, "rows": x2[idx].clone(), "sum": float(x2.double().sum()), "abs_sum": float(x2.double().abs().sum())}


def nav_bev():
    """nav_bev.pt: the agents' BEV input over a synthetic episode (tests/nav_bev_cases.py), from the reference's own
    GraphMap (map_nav_src/models/graph_utils.py) and PointCloud.project_bev (map_nav_src/models/bev_utils.py, through
    ref_shim's scatter_mean), with the ego transform of agent.py:150-166.  Per step and sample: the viewpoints
    gather_node_pc concatenated (recovered from its output), the node_pc key order and path lengths it chose from,
    the reference's cell index of the concatenated cloud and its pooled map (per-cell float64 sums, a row sample,
    ob_mask)."""
    import numpy as np
    from torch.nn.utils.rnn import pad_sequence
    import nav_bev_cases as NB
    ref_shim.load_pretrain_modules()                   # installs the torch_scatter stub
    src = os.path.join(ref_shim.REF_ROOT, "map_nav_src")
    if src not in sys.path:
        sys.path.insert(0, src)
    import importlib
    graph_utils = importlib.import_module("models.graph_utils")
    bev_utils = importlib.import_module("models.bev_utils")
    D, res, B = 21, 0.5, 3
    projector = bev_utils.PointCloud(np.radians(90), 1, feature_map_height=14, feature_map_width=14, map_dim=D,
                                     map_res=res, world_shift_origin=torch.zeros(3), z_clip_threshold=0.5,
                                     device=torch.device("cpu"))
    ep = NB.episode(B=B)
    gmaps = [graph_utils.GraphMap(ep[0][0][i]["viewpoint"]) for i in range(B)]
    steps = []
    for t, (obs, clouds, order) in enumerate(ep):
        rec = {"order": order, "vps": [], "keys": [], "hops": [], "cell_idx": []}
        pcs, masks, feats = [], [], []
        for i, (ob, gm) in enumerate(zip(obs, gmaps)):
            gm.update_graph(ob)
            gm.update_node_pc(ob["viewpoint"], *clouds[i])
            pc, m, f = gm.gather_node_pc(ob["viewpoint"], order)
            vps, o = [], 0
            while o < pc.shape[0]:
                k = next(k for k, v in gm.node_pc.items() if o + v[0].shape[0] <= pc.shape[0] and torch.equal(pc[o:o + v[0].shape[0]], v[0]))
                vps.append(k)
                o += gm.node_pc[k][0].shape[0]
            rec["vps"].append(vps)
            rec["keys"].append(list(gm.node_pc.keys()))
            rec["hops"].append([len(gm.graph.path(ob["viewpoint"], k)) for k in gm.node_pc])
            pcs.append(pc)
            masks.append(m)
            feats.append(f)
        pc = pad_sequence(pcs, batch_first=True)
        mask = pad_sequence(masks, batch_first=True, padding_value=True)
        feat = pad_sequence(feats, batch_first=True)
        S = torch.from_numpy(np.vstack([[np.array([o["position"][0], o["position"][2], -o["position"][1]])]
                                        for o in obs]).astype(np.float32))
        xyzhe = np.zeros([B, 5])
        xyzhe[:, 3] = [o["heading"] for o in obs]
        T = torch.from_numpy(bev_utils.transfrom3D(xyzhe))
        pc = pc - S[:, None, :]
        pc1 = torch.matmul(torch.cat([pc, torch.ones(pc.shape[:2]).unsqueeze(-1)], -1), T.transpose(1, 2))
        bev, ob = projector.project_bev(pc1[:, :, :3], mask, feat)
        idx = cell_index(pc1[:, :, :3], mask, D, res)
        rec["cell_idx"] = [idx[i, :pcs[i].shape[0]].to(torch.int16).clone() for i in range(B)]
        bev = bev.reshape(B, D * D, -1)
        rec["cell_sums"] = bev.double().sum(-1)
        rec["bev"] = sample_rows(bev, 4, t)
        rec["ob_masks"] = ob.reshape(B, -1).clone()
        steps.append(rec)
        print("nav_bev step", t, "order", order, "nodes", [len(v) for v in rec["vps"]])
    torch.save({"D": D, "res": res, "B": B, "steps": steps},
               os.path.join(os.path.dirname(os.path.abspath(__file__)), "nav_bev.pt"))



if __name__ == "__main__":
    nav_bev()
