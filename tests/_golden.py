"""Golden fixtures on disk: every file stays under 1 MB, so the network weights (`state`) of a fixture are stored in a
file of their own and the main file holds that file's name in their place."""
import os

import torch

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")


def load(name):
    g = torch.load(os.path.join(GOLDEN, name), weights_only=True)
    for v in g.values():
        if isinstance(v, dict) and isinstance(v.get("state"), str):
            v["state"] = torch.load(os.path.join(GOLDEN, v["state"]), weights_only=True)
    return g


def save(g, name):
    base = name[:-3]
    out = {}
    for k, v in g.items():
        if isinstance(v, dict) and isinstance(v.get("state"), dict):
            sname = "%s_%s_state.pt" % (base, k)
            torch.save(v["state"], os.path.join(GOLDEN, sname))
            v = dict(v, state=sname)
        out[k] = v
    torch.save(out, os.path.join(GOLDEN, name))
