"""Float64 restatement of the sky model (scene/background_model.py SkyModel + get_directions, scene/encodings.py
SinusoidalEncoder) and of its weight gradients, for the tests.

directions(c2w, K, H, W) -> v [H*W, 3]; encode(v) -> [H*W, 33]; sky64(params, c2w, K, H, W) -> [3, H, W] through
autograd; sky_grads64 gives the output and every parameter gradient in closed form, in pixel chunks, so that it runs
at 1920 x 1280 without autograd's activations.  params = (W0, b0, W1, b1, W2, b2) in nn.Linear's layout."""
import math

import torch

SCALES = (1.0, 2.0, 4.0, 8.0, 16.0)


def directions(c2w, K, H, W, pix=None):
    c2w, K = c2w.double(), K.double()
    dev = c2w.device
    if pix is None:
        pix = torch.arange(H * W, device=dev)
    x, y = (pix % W).double(), (pix // W).double()
    cam = torch.stack([(x - K[0, 2] + 0.5) / K[0, 0], (y - K[1, 2] + 0.5) / K[1, 1], torch.ones_like(x)], -1)
    d = cam @ c2w[:3, :3].T
    return d / (d.norm(dim=-1, keepdim=True) + 1e-8)


def encode(v):
    xb = torch.cat([v * s for s in SCALES], -1)               # scale-major, 3 values per scale
    return torch.cat([v, torch.sin(xb), torch.sin(xb + 0.5 * math.pi)], -1)


def sky64(params, c2w, K, H, W):
    W0, b0, W1, b1, W2, b2 = params
    e = encode(directions(c2w, K, H, W)).to(W0.dtype)
    h1 = torch.relu(e @ W0.T + b0)
    h2 = torch.relu(torch.cat([h1, e], -1) @ W1.T + b1)
    return torch.sigmoid(h2 @ W2.T + b2).T.reshape(3, H, W)


def sky_grads64(params, c2w, K, H, W, gsky=None, chunk=1 << 16):
    """(sky [3,H,W], grads of (W0, b0, W1, b1, W2, b2) for the upstream gsky [3,H,W]) in float64 on params' device."""
    W0, b0, W1, b1, W2, b2 = (p.double() for p in params)
    dev = W0.device
    out = torch.empty(3, H * W, dtype=torch.float64, device=dev)
    grads = [torch.zeros_like(p) for p in (W0, b0, W1, b1, W2, b2)]
    g = None if gsky is None else gsky.double().reshape(3, H * W).to(dev)
    Wd = W0.shape[0]
    for p0 in range(0, H * W, chunk):
        pix = torch.arange(p0, min(H * W, p0 + chunk), device=dev)
        e = encode(directions(c2w.to(dev), K.to(dev), H, W, pix))
        h1 = torch.relu(e @ W0.T + b0)
        x1 = torch.cat([h1, e], -1)
        h2 = torch.relu(x1 @ W1.T + b1)
        s = torch.sigmoid(h2 @ W2.T + b2)
        out[:, pix] = s.T
        if g is None:
            continue
        dz = g[:, pix].T * s * (1 - s)
        grads[4] += dz.T @ h2
        grads[5] += dz.sum(0)
        d2 = (dz @ W2) * (h2 > 0)
        grads[2] += d2.T @ x1
        grads[3] += d2.sum(0)
        d1 = (d2 @ W1[:, :Wd]) * (h1 > 0)
        grads[0] += d1.T @ e
        grads[1] += d1.sum(0)
    return out.reshape(3, H, W), grads
