"""Generate tests/golden/step_glue.pt from the UNMODIFIED reference host-glue functions (run in this container only):

    python tests/golden/make_glue_golden.py

A synthetic 3-episode, 5-step rollout on a random viewpoint graph is pushed through the reference's
GraphMap / FloydGraph (models/graph_utils.py:46-165) and MP3DAgent.panorama_feature_variable_object / nav_vp_variable /
nav_gmap_variable (tasks/agents/mp3d_agent.py:143-212, 264-371) with torch.Tensor.cuda patched to the identity (no GPU here).
The observations and every returned tensor / list are stored; tests/test_step_glue_cpu.py replays the observations through
navillm_b200.step_glue and compares.
"""
import os
import sys
import types
from pathlib import Path

import numpy as np
import torch

sys.path.insert(0, os.environ["NAVILLM_REFERENCE"])   # a checkout of the reference
torch.Tensor.cuda = lambda self, *a, **k: self          # the reference calls .cuda() on everything it builds

from models.graph_utils import GraphMap  # noqa: E402
from tasks.agents.mp3d_agent import MP3DAgent  # noqa: E402

F, A, D = 16, 4, 32


def make_world(rng, n=14):
    pos = {f"vp{i}": (float(rng.uniform(-8, 8)), float(rng.uniform(-8, 8)), float(rng.uniform(-1, 1))) for i in range(n)}
    names = list(pos)
    adj = {v: set() for v in names}
    for i, v in enumerate(names):                       # ring + a few chords: connected, degree 2..5
        for w in (names[(i + 1) % n], names[(i + 3) % n] if i % 2 == 0 else None):
            if w is not None and w != v:
                adj[v].add(w); adj[w].add(v)
    return pos, {v: sorted(a) for v, a in adj.items()}


def make_ob(rng, pos, adj, vp, heading, with_obj):
    feats = rng.randn(36, F + A).astype(np.float32)
    cands = []
    for j, w in enumerate(adj[vp]):
        cands.append({"viewpointId": w, "pointId": int(3 * j + 1), "feature": rng.randn(F + A).astype(np.float32), "position": pos[w]})
    ob = {"viewpoint": vp, "heading": heading, "elevation": 0.0, "position": pos[vp], "candidate": cands, "feature": list(feats)}
    if with_obj:
        n = int(rng.randint(2, 6))
        ob.update({"obj_img_fts": rng.randn(n, 12).astype(np.float32), "obj_ang_fts": rng.randn(n, 4).astype(np.float32),
                   "obj_box_fts": rng.rand(n, 3).astype(np.float32), "obj_ids": [f"o{k}" for k in range(n)]})
    return ob


def main():
    rng = np.random.RandomState(7)
    g = torch.Generator().manual_seed(7)
    pos, adj = make_world(rng)
    B, STEPS = 3, 5
    cur = ["vp0", "vp5", "vp9"]
    fake = types.SimpleNamespace(args=types.SimpleNamespace(image_feat_size=F, enc_full_graph=True))
    gmaps = [GraphMap(v) for v in cur]
    steps = []
    for t in range(STEPS):
        obs = [make_ob(rng, pos, adj, cur[i], heading=float(rng.uniform(0, 6.28)), with_obj=(t == 2)) for i in range(B)]
        for i, gm in enumerate(gmaps):
            gm.update_graph(obs[i])
            gm.node_step_ids[obs[i]["viewpoint"]] = t + 1
        pano_in = MP3DAgent.panorama_feature_variable_object(fake, obs)
        NV = pano_in["view_img_fts"].shape[1]
        pano_embeds = torch.randn(B, NV, D, generator=g)
        pano_masks = torch.arange(NV)[None, :] < pano_in["view_lens"][:, None]
        avg = (pano_embeds * pano_masks.unsqueeze(2)).sum(1) / pano_masks.sum(1, keepdim=True)
        for i, gm in enumerate(gmaps):                                  # tasks/agents/mp3d_agent.py:690-700
            gm.update_node_embed(obs[i]["viewpoint"], avg[i].clone(), rewrite=True)
            for j, cv in enumerate(pano_in["cand_vpids"][i]):
                if not gm.graph.visited(cv):
                    gm.update_node_embed(cv, pano_embeds[i, j].clone())
        nav = MP3DAgent.nav_gmap_variable(fake, obs, gmaps)
        nav.update(MP3DAgent.nav_vp_variable(fake, obs, gmaps, pano_embeds, pano_masks, pano_in["cand_vpids"], pano_in["view_lens"],
                                             pano_in["nav_types"]))
        steps.append({"obs": obs, "pano_in": pano_in, "pano_embeds": pano_embeds, "pano_masks": pano_masks, "nav": nav})
        # move: first unvisited candidate if any, else first candidate
        for i, gm in enumerate(gmaps):
            nxt = [c["viewpointId"] for c in obs[i]["candidate"] if not gm.graph.visited(c["viewpointId"])]
            cur[i] = nxt[0] if nxt else obs[i]["candidate"][0]["viewpointId"]
    out = Path(__file__).with_name("step_glue.pt")
    torch.save({"F": F, "A": A, "D": D, "start": ["vp0", "vp5", "vp9"], "steps": steps}, out)
    print("wrote", out, out.stat().st_size, "bytes")


if __name__ == "__main__":
    main()
