"""Float64 restatement of ``ConditionalDiscriminator.forward`` (model/vtoonify.py:10-89) from oracle/vt_oracle.py's pieces and a
conv2d, on a state_dict.  Parametrised by the three ops (``conv2d``, ``upfirdn2d``, ``fused_leaky_relu``) like ``_discriminator`` in
tests/test_gpu_conv_grad.py, so the same statements are the fixtures' checker (float64 on the CPU), the cuDNN arm and the
``vtoonify_b200.op`` arm of tools/discriminator_bench.py.  Differentiable: every piece is torch autograd."""
import math

import torch
import torch.nn.functional as F

from oracle import vt_oracle as O

CASES = {"cond": dict(use_condition=True, style_num=5), "plain": dict(use_condition=False)}
SIZE, CHANNEL_MULTIPLIER, BATCH = 64, 1, 8
WSTEP = 401


def _eq(w):
    return w * (1 / math.sqrt(w[0].numel()))


def n_blocks(sd):
    return sum(1 for k in sd if k.startswith("convs.") and k.endswith(".conv1.0.weight"))


def trunk(sd, x, conv2d=F.conv2d, upfirdn2d=O.upfirdn2d, flrelu=O.fused_leaky_relu):
    """``convs``: ConvLayer(3, C, 1), then the ResBlocks."""
    K = O.make_kernel([1, 3, 3, 1]).to(x)
    h = flrelu(conv2d(x, _eq(sd["convs.0.0.weight"]), None, stride=1, padding=0), sd["convs.0.1.bias"])
    for i in range(1, n_blocks(sd) + 1):
        p = f"convs.{i}."
        o = flrelu(conv2d(h, _eq(sd[p + "conv1.0.weight"]), None, stride=1, padding=1), sd[p + "conv1.1.bias"])
        o = flrelu(conv2d(upfirdn2d(o, K, pad=(2, 2)), _eq(sd[p + "conv2.1.weight"]), None, stride=2, padding=0), sd[p + "conv2.2.bias"])
        sk = conv2d(upfirdn2d(h, K, pad=(1, 1)), _eq(sd[p + "skip.1.weight"]), None, stride=2, padding=0)
        h = (o + sk) / math.sqrt(2)
    return h


def mbstd(out, group_size=4):
    """model/vtoonify.py:67-75"""
    batch, channel, height, width = out.shape
    group = min(batch, group_size)
    stddev = out.view(group, -1, 1, channel, height, width)
    stddev = torch.sqrt(stddev.var(0, unbiased=False) + 1e-8)
    stddev = stddev.mean([2, 3, 4], keepdims=True).squeeze(2)
    stddev = stddev.repeat(group, 1, height, width)
    return torch.cat([out, stddev], 1)


def head(sd, h, conv2d=F.conv2d, flrelu=O.fused_leaky_relu):
    """minibatch stddev, final_conv, final_linear -> [B, condition_dim]"""
    out = flrelu(conv2d(mbstd(h), _eq(sd["final_conv.0.weight"]), None, stride=1, padding=1), sd["final_conv.1.bias"])
    out = out.reshape(out.shape[0], -1)
    out = O.equal_linear(out, sd["final_linear.0.weight"], sd["final_linear.0.bias"], activation=True)
    return O.equal_linear(out, sd["final_linear.1.weight"], sd["final_linear.1.bias"])


def condition(sd, h, degree_label, style_ind):
    lm = degree_label
    for i in (0, 2, 4):
        lm = F.linear(lm, sd[f"label_mapper.{i}.weight"], sd[f"label_mapper.{i}.bias"])
        if i < 4:
            lm = F.leaky_relu(lm, 0.2)
    cond = torch.cat((lm, F.embedding(style_ind, sd["style_mapper.weight"])), dim=1)
    return (h * cond).sum(dim=1, keepdim=True) * (1 / math.sqrt(h.shape[1]))


def forward(sd, x, degree_label=None, style_ind=None, **ops):
    conv2d = ops.get("conv2d", F.conv2d)
    flrelu = ops.get("flrelu", O.fused_leaky_relu)
    h = head(sd, trunk(sd, x, conv2d, ops.get("upfirdn2d", O.upfirdn2d), flrelu), conv2d, flrelu)
    if "style_mapper.weight" in sd:
        return condition(sd, h, degree_label, style_ind)
    return h


def case_inputs(case, B=BATCH, size=SIZE, seed=7):
    """Seeded image, degree labels and style indices of a fixture case."""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn((B, 3, size, size), generator=g)
    d = torch.rand((B, 1), generator=g)
    s = torch.randint(0, CASES[case].get("style_num") or 1, (B,), generator=g)
    return x, d, s


def loss_fn(out):
    """``softplus(-out).mean()``: the generator's non-saturating loss"""
    return F.softplus(-out).mean()
