#!/usr/bin/env python
"""Generate tests/golden/tiling_tiny.npz by running the REAL reference on CPU with wrap-around padding.

Needs a reference checkout, found and loaded as make_golden.py finds and loads it ($PAELLA_REFERENCE):
    python tests/golden/make_golden_tiling.py
The inputs and weights are those of the committed paella_tiny.npz and vqgan_tiny.npz; only the padding of the reference
modules changes, by the users' idiom (padding_mode='circular' on Conv2d) or by wrapping a module around the same weights.
"""
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)

from make_golden import TINY, TINY_VQ, load_reference     # noqa: E402


class _AxisPad(torch.nn.Module):
    """Pad one position per side: circularly on the wrapped axes, with ``fill`` ('constant' zeros or 'replicate') elsewhere."""

    def __init__(self, p, wrap_x, wrap_y, fill):
        super().__init__()
        self.p, self.wrap_x, self.wrap_y, self.fill = p, wrap_x, wrap_y, fill

    def forward(self, x):
        p = self.p
        x = torch.nn.functional.pad(x, (0, 0, p, p), mode="circular" if self.wrap_y else self.fill)
        return torch.nn.functional.pad(x, (p, p, 0, 0), mode="circular" if self.wrap_x else self.fill)


class _PaddedConv(torch.nn.Module):
    """The same conv weights run with padding 0 after an _AxisPad, then cropped by ``crop`` on every side."""

    def __init__(self, conv, pad, crop=0):
        super().__init__()
        self.conv, self.pad, self.crop = conv, pad, crop
        conv.padding = (0, 0)

    def forward(self, x, *a):
        y = self.conv(self.pad(x))
        c = self.crop
        return y[..., c:y.shape[-2] - c, c:y.shape[-1] - c] if c else y


def tiling():
    """tests/golden/tiling_tiny.npz: the reference's tiny denoiser and tiny codec with wrap-around padding, on the inputs of
    paella_tiny.npz / vqgan_tiny.npz.  'xy' is the users' idiom, padding_mode='circular' on every Conv2d of the denoiser; 'x'
    and 'y' wrap each ResBlock depthwise conv in a module that pads one axis circularly and the other with zeros.  The codec
    swaps each ReplicationPad2d for the circular pad and runs its ConvTranspose2d(k4, s2, p1) as a circular pad of 1, the conv
    with padding 0 and a crop of 3 per side (an unwrapped axis is padded with zeros, which adds nothing)."""
    torch.set_grad_enabled(False)
    _, ref_nb_modules, _, ref_vqgan, _ = load_reference()
    _, psd, pg = (lambda z: (None, {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")},
                             {k: z[k] for k in z.files}))(np.load(os.path.join(HERE, "paella_tiny.npz")))
    x, r = torch.from_numpy(pg["x"]), torch.from_numpy(pg["r"])
    byt5, clip, clip_image = (torch.from_numpy(pg[k]) for k in ("byt5", "clip", "clip_image"))
    out = {}
    for name, (wx, wy) in (("xy", (True, True)), ("x", (True, False)), ("y", (False, True))):
        torch.manual_seed(0)
        m = ref_nb_modules.Paella(**TINY).eval()
        m.load_state_dict(psd)
        if name == "xy":
            for mod in m.modules():
                if isinstance(mod, torch.nn.Conv2d):
                    mod.padding_mode = "circular"
        else:
            for mod in m.modules():
                if isinstance(mod, ref_nb_modules.ResBlock):
                    k = mod.depthwise.kernel_size[0]
                    mod.depthwise = _PaddedConv(mod.depthwise, _AxisPad(k // 2, wx, wy, "constant"))
        out["logits_" + name] = m(x, r, byt5, clip=clip, clip_image=clip_image).numpy()
    z = np.load(os.path.join(HERE, "vqgan_tiny.npz"))
    vsd = {k[3:]: torch.from_numpy(z[k]) for k in z.files if k.startswith("sd:")}
    idx = torch.from_numpy(z["idx_rand"])
    out["idx"] = idx.numpy()
    for name, (wx, wy) in (("xy", (True, True)), ("x", (True, False))):
        torch.manual_seed(3)
        vq = ref_vqgan.VQModel(**TINY_VQ).eval()
        vq.load_state_dict(vsd)
        for mod in list(vq.modules()):
            for cname, child in list(mod.named_children()):
                if isinstance(child, torch.nn.ReplicationPad2d):
                    setattr(mod, cname, _AxisPad(1, wx, wy, "replicate"))
                elif isinstance(child, torch.nn.ConvTranspose2d):
                    setattr(mod, cname, _PaddedConv(child, _AxisPad(1, wx, wy, "constant"), crop=3))
        out["dec_" + name] = vq.decode_indices(idx).numpy()
    np.savez_compressed(os.path.join(HERE, "tiling_tiny.npz"), **out)
    print("tiling_tiny.npz:", {k: v.shape for k, v in out.items()})


if __name__ == "__main__":
    tiling()
