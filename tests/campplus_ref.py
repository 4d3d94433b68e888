"""Float64 restatement of CAMPPlus.forward (funasr/models/campplus/model.py, components.py) in eval mode on the CPU, and the
per-utterance metric the CAM++ parity tests use.  Pinned to the reference by tests/test_campplus_host.py: against the embeddings the
reference stored in the fixtures (cb_in) and, where the reference tree is present, against its CAMPPlus class run live."""
import numpy as np
import torch
import torch.nn.functional as F


def _bn(sd, p, x, dim=1):
    shape = [1] * x.dim()
    shape[dim] = -1
    y = (x - sd[p + ".running_mean"].double().view(shape)) / torch.sqrt(sd[p + ".running_var"].double().view(shape) + 1e-5)
    if (p + ".weight") in sd:
        y = y * sd[p + ".weight"].double().view(shape) + sd[p + ".bias"].double().view(shape)
    return y


def cam_layer_ref(h, wl, w1, b1, w2, b2, dil):
    """CAMLayer.forward on h [B, C, T] (float64)."""
    y = F.conv1d(h, wl, padding=dil, dilation=dil)
    T = h.shape[-1]
    seg = F.avg_pool1d(h, kernel_size=100, stride=100, ceil_mode=True)
    seg = seg.unsqueeze(-1).expand(*seg.shape, 100).reshape(*seg.shape[:-1], -1)[..., :T]
    ctx = h.mean(-1, keepdim=True) + seg
    m = torch.sigmoid(F.conv1d(F.relu(F.conv1d(ctx, w1, b1)), w2, b2))
    return y * m


def campplus_ref(sd, feats):
    """CAMPPlus.forward (eval) in float64 on the CPU: feats [B, T, 80] -> [B, 192].  At T = 2 (one TDNN frame) the unbiased std of
    the statistics pooling is 0 / 0 and every output is NaN, as in the reference."""
    sd = {k: v.double() if v.is_floating_point() else v for k, v in sd.items()}
    x = feats.double().permute(0, 2, 1).unsqueeze(1)

    def conv_bn(x, conv, bn, stride=1, pad=1):
        return _bn(sd, "head." + bn, F.conv2d(x, sd["head." + conv + ".weight"], stride=(stride, 1), padding=pad))

    x = F.relu(conv_bn(x, "conv1", "bn1"))
    for layer in ("layer1", "layer2"):
        for b in (0, 1):
            p = "%s.%d." % (layer, b)
            s = 2 if b == 0 else 1
            out = F.relu(conv_bn(x, p + "conv1", p + "bn1", s))
            out = conv_bn(out, p + "conv2", p + "bn2")
            sc = conv_bn(x, p + "shortcut.0", p + "shortcut.1", s, 0) if b == 0 else x
            x = F.relu(out + sc)
    x = F.relu(conv_bn(x, "conv2", "bn2", 2))
    x = x.reshape(x.shape[0], -1, x.shape[-1])
    x = F.relu(_bn(sd, "xvector.tdnn.nonlinear.batchnorm", F.conv1d(x, sd["xvector.tdnn.linear.weight"], stride=2, padding=2)))
    for i, (n, dil) in enumerate(zip((12, 24, 16), (1, 2, 2))):
        for l in range(n):
            p = "xvector.block%d.tdnnd%d." % (i + 1, l + 1)
            h = F.conv1d(F.relu(_bn(sd, p + "nonlinear1.batchnorm", x)), sd[p + "linear1.weight"])
            h = F.relu(_bn(sd, p + "nonlinear2.batchnorm", h))
            y = cam_layer_ref(h, sd[p + "cam_layer.linear_local.weight"], sd[p + "cam_layer.linear1.weight"], sd[p + "cam_layer.linear1.bias"],
                              sd[p + "cam_layer.linear2.weight"], sd[p + "cam_layer.linear2.bias"], dil)
            x = torch.cat([x, y], 1)
        p = "xvector.transit%d." % (i + 1)
        x = F.conv1d(F.relu(_bn(sd, p + "nonlinear.batchnorm", x)), sd[p + "linear.weight"])
    x = F.relu(_bn(sd, "xvector.out_nonlinear.batchnorm", x))
    x = torch.cat([x.mean(-1), x.std(-1, unbiased=True)], -1)
    return _bn(sd, "xvector.dense.nonlinear.batchnorm", F.conv1d(x.unsqueeze(-1), sd["xvector.dense.linear.weight"]).squeeze(-1))


def emb_err(got, ref):
    """Per utterance of [B, 192] embeddings -> (max_c |got - ref| / max_c |ref|, 1 - cos(got, ref)), both float64 [B]."""
    g = np.asarray(torch.as_tensor(got).detach().cpu().double())
    r = np.asarray(torch.as_tensor(ref).detach().cpu().double())
    rel = np.abs(g - r).max(-1) / np.abs(r).max(-1)
    cos = (g * r).sum(-1) / (np.linalg.norm(g, axis=-1) * np.linalg.norm(r, axis=-1))
    return rel, 1.0 - cos
