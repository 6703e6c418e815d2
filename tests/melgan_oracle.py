"""CPU oracle of MelGAN.forward (models/vocoders/gan/generator/melgan.py:50-101) on a reference state dict:
CPU torch fp32, weight norm folded as torch does, reflection padding included."""
import numpy as np
import torch
import torch.nn.functional as F

# hyper-parameters of tests/golden/melgan.npz (tests/golden/gen_melgan.py): tag -> (melgan hp, n_mel, B, T)
GOLDEN_MELGAN = {
    "a": (dict(ratios=[4, 2], ngf=16, n_residual_layers=3), 20, 2, 24),
    "b": (dict(ratios=[3, 5], ngf=8, n_residual_layers=2), 12, 1, 7),
}
# egs/vocoder/gan/melgan/exp_config.json with exp_config_base.json's 100 mels
HP_MELGAN_RECIPE = dict(ratios=[8, 8, 2, 2], ngf=32, n_residual_layers=3)


def _t(v):
    return torch.as_tensor(np.asarray(v), dtype=torch.float32)


def _weight(params, name):
    if name + ".weight" in params:
        return _t(params[name + ".weight"])
    return torch._weight_norm(_t(params[name + ".weight_v"]), _t(params[name + ".weight_g"]), 0)


def melgan_forward(params, hp, mel, stages=False):
    """mel [B, n_mel, T] -> wav [B, 1, T * prod(ratios)] (numpy fp32); with ``stages`` also the output of every
    stage's last ResnetBlock."""
    R, n = int(hp["n_residual_layers"]), len(hp["ratios"])

    def conv(x, i, **kw):
        name = f"model.{i}"
        return F.conv1d(x, _weight(params, name), _t(params[name + ".bias"]), **kw)

    outs = []
    with torch.no_grad():
        x = conv(F.pad(_t(mel), (3, 3), mode="reflect"), 1)
        for i, r in enumerate(hp["ratios"]):
            base = 2 + i * (2 + R)
            name = f"model.{base + 1}"
            x = F.conv_transpose1d(F.leaky_relu(x, 0.2), _weight(params, name), _t(params[name + ".bias"]), stride=r,
                                   padding=r // 2 + r % 2, output_padding=r % 2)
            for j in range(R):
                d, blk = 3 ** j, base + 2 + j
                h = F.pad(F.leaky_relu(x, 0.2), (d, d), mode="reflect")
                h = conv(h, f"{blk}.block.2", dilation=d)
                h = conv(F.leaky_relu(h, 0.2), f"{blk}.block.4")
                x = conv(x, f"{blk}.shortcut") + h
            outs.append(x.numpy())
        x = F.pad(F.leaky_relu(x, 0.2), (3, 3), mode="reflect")
        y = torch.tanh(conv(x, 2 + n * (2 + R) + 2)).numpy()
    return (y, outs) if stages else y
