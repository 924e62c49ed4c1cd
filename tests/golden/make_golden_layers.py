"""Per-LAYER golden vectors: forward hooks on the UNMODIFIED reference networks, keyed like the oracle's `trace=` checkpoints
(which the GPU per-layer parity reports compare against).  Pins the oracle's per-layer restatement, not only its output.

    python tests/golden/make_golden_layers.py        # needs /root/reference; writes reference_golden_layers.pt

Reference modules hooked (codes/config/{deraining,denoising-sde}/models/modules/DenoisingUNet_arch.py, module_util.py):
  init_conv, every Block `block1` (module_util.py:55-67), every conv `res_conv`, every ResBlock (:108-146), every PreNorm's
  LayerNorm (:70-90), LinearAttention.to_out[0] (:159-178), every Residual(PreNorm(attention)) (:20-26), Downsample /
  Upsample convs (:93-101), the input of Attention.to_out (:190-204)."""
import importlib
import os
import sys
import types

import torch


def load(task):
    ref = "/root/reference/codes/config/%s/models/modules" % task
    name = "refpkg_layers_" + task.replace("-", "_")
    pkg = types.ModuleType(name)
    pkg.__path__ = [ref]
    sys.modules[name] = pkg
    return importlib.import_module(name + ".DenoisingUNet_arch")


def fingerprint(t):
    """What is stored per layer (keeps the fixture small): shape, fp64 sum and abs-sum, and <= 512 evenly strided elements."""
    f = t.detach().reshape(-1)
    stride = max(1, f.numel() // 512)
    return {"shape": torch.tensor(list(t.shape)), "sum": f.double().sum(), "abssum": f.double().abs().sum(),
            "stride": torch.tensor(stride), "sample": f[::stride].clone()}


def hooked_forward(net, run):
    """{oracle trace key: fingerprint} from forward hooks on the reference module tree."""
    layers = {}
    hooks = []

    def out_hook(key):
        return lambda mod, inp, out: layers.__setitem__(key, fingerprint(out))

    def in_hook(key):
        return lambda mod, inp: layers.__setitem__(key, fingerprint(inp[0]))

    for name, mod in net.named_modules():
        cls = type(mod).__name__
        if name == "init_conv":
            hooks.append(mod.register_forward_hook(out_hook("init_conv.weight")))
        elif cls == "Block" and name.endswith("block1"):
            hooks.append(mod.register_forward_hook(out_hook(name + ".proj.weight")))
        elif name.endswith("res_conv") and isinstance(mod, torch.nn.Conv2d):
            hooks.append(mod.register_forward_hook(out_hook(name + ".weight")))
        elif cls == "ResBlock":
            hooks.append(mod.register_forward_hook(out_hook(name + ".block2.proj.weight")))
        elif cls == "LayerNorm" and name.endswith(".fn.norm"):
            hooks.append(mod.register_forward_hook(out_hook(name[:-len("fn.norm")] + "norm")))
        elif cls == "LinearAttention":
            hooks.append(mod.to_out[0].register_forward_hook(out_hook(name + ".to_out.0.weight")))
        elif cls == "Attention":
            base = name[:-len("fn.fn")]
            hooks.append(mod.to_out.register_forward_pre_hook(in_hook(base + "full attention")))
        elif cls == "Residual":
            inner = type(mod.fn.fn).__name__
            key = name + ".to_out.norm+res" if inner == "LinearAttention" else name + ".fn.fn.to_out.weight"
            hooks.append(mod.register_forward_hook(out_hook(key)))
        elif isinstance(mod, torch.nn.Conv2d) and (name.split(".")[0] in ("downs", "ups")) and name.split(".")[2:3] == ["3"]:
            hooks.append(mod.register_forward_hook(out_hook(name + ".weight")))
    with torch.no_grad():
        y = run(net)
    for h in hooks:
        h.remove()
    return layers, y


def randomise(net, seed):
    torch.manual_seed(seed)
    with torch.no_grad():
        for n, p in net.named_parameters():   # non-trivial gains / biases (the constructors leave g = 1)
            if n.endswith(".g"):
                p.add_(0.1 * torch.randn_like(p))


out = {}
g = torch.Generator().manual_seed(11)
# conditional UNet (deraining), ragged input -> reflect pad
arch = load("deraining")
torch.manual_seed(0)
cfg = dict(in_nc=3, out_nc=3, nf=8, depth=2)
net = arch.ConditionalUNet(**cfg).eval()
randomise(net, 1)
x, c = torch.rand(2, 3, 18, 26, generator=g), torch.rand(2, 3, 18, 26, generator=g)
layers, y = hooked_forward(net, lambda m: m(x, c, 7))
out["cond"] = {"cfg": cfg, "state": {k: v.detach().clone() for k, v in net.state_dict().items()}, "x": x, "cond": c, "t": 7,
               "y": y, "layers": layers}
# denoising-sde variant (full softmax Attention at mid_attn)
arch = load("denoising-sde")
torch.manual_seed(2)
cfg = dict(in_nc=3, out_nc=3, nf=8, depth=2)
net = arch.ConditionalUNet(**cfg).eval()
randomise(net, 3)
x = torch.rand(2, 3, 16, 24, generator=g)
layers, y = hooked_forward(net, lambda m: m(x, 5))
out["denoising"] = {"cfg": cfg, "state": {k: v.detach().clone() for k, v in net.state_dict().items()}, "x": x, "t": 5, "y": y,
                    "layers": layers}
sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), ".."))
import _golden  # noqa: E402
_golden.save(out, "reference_golden_layers.pt")
for k, v in out.items():
    print(k, len(v["layers"]), "layers", float(v["y"].abs().max()))
