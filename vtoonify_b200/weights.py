"""Deterministic synthetic weights (there are no checkpoints offline): every tensor of a state_dict is drawn from a
CPU generator seeded by crc32(key) ^ seed, with per-key scales chosen so activations stay O(1) through ~50 stacked
convolutions and the output image is O(0.5) (the range of a trained model), which makes absolute-error bars meaningful.
The same function seeds the reference model (tests/golden/make_golden.py), the oracle and the CUDA modules, so parity
runs share bit-identical parameters without shipping 650 MB of weights."""
import math
import re
import zlib

import torch


# top-level keys of a ConditionalDiscriminator state_dict that hold an EqualConv2d / EqualLinear weight (no other model's keys match)
DISCRIMINATOR_EQUAL_WEIGHT = re.compile(r"^(convs\.\d+\.(0|conv1\.0|conv2\.1|skip\.1)|final_conv\.0|final_linear\.\d)\.weight$")


def det_tensor(key: str, ref: torch.Tensor, seed: int = 0) -> torch.Tensor:
    shape = tuple(ref.shape)
    g = torch.Generator(device="cpu")
    g.manual_seed((zlib.crc32(key.encode()) ^ (seed * 0x9E3779B1)) & 0x7FFFFFFF)
    r = torch.randn(shape, generator=g, dtype=torch.float32)
    if key.endswith("num_batches_tracked"):
        return torch.zeros(shape, dtype=torch.long)
    if key.endswith("running_var"):
        return 0.5 + torch.rand(shape, generator=g)
    if key.endswith("running_mean"):
        return 0.1 * r
    if ref.dim() == 1 and re.search(r"res_layer\.4\.weight$", key):
        return 0.2 * (1.0 + 0.1 * r)                            # last BN of a residual branch: small gamma keeps the 24-block
                                                                 # IR stack well conditioned (gamma ~ 1 makes it chaotic: a 1e-7
                                                                 # perturbation grows 1.8x per block, measured)
    if ref.dim() == 1 and re.search(r"(^|\.)bn2\.weight$", key):
        return 0.5 * (1.0 + 0.1 * r)                            # BiSeNet / ResNet-18: last BN of a residual branch
    if ref.dim() == 1 and re.search(r"(^|\.)(bn\d*|bn_atten|downsample\.1)\.weight$", key):
        return 1.0 + 0.1 * r                                    # BiSeNet BatchNorm gamma
    if ref.dim() == 1 and re.search(r"(input_layer\.1|res_layer\.0|shortcut_layer\.1)\.weight$", key):
        return 1.0 + 0.1 * r                                    # BatchNorm gamma
    if ref.dim() == 1 and re.search(r"(input_layer\.2|res_layer\.2)\.weight$", key):
        return 0.25 + 0.05 * r                                   # PReLU slopes
    if key.endswith("blur.kernel") or key.endswith("upsample.kernel") or key.endswith(".0.kernel"):
        return ref.detach().clone().float()                      # FIR taps are architecture constants
    if DISCRIMINATOR_EQUAL_WEIGHT.search(key):
        return r                                                 # ConditionalDiscriminator's EqualConv2d / EqualLinear weights:
                                                                 # randn, as the reference initialises them (the layer's own
                                                                 # 1/sqrt(fan_in) keeps activations O(1))
    if "noises.noise_" in key or key.endswith("input.input"):
        return r
    if key.endswith("modulation.weight"):
        return r
    if key.endswith("modulation.bias"):
        return 1.0 + 0.1 * r
    if key.endswith("noise.weight"):
        return 0.1 * r
    if re.search(r"(^|\.)style\.\d+\.weight$", key) and ref.dim() == 2 and shape[0] == shape[1]:
        return r / 0.01                                          # EqualLinear(lr_mul=0.01): weight = randn / lr_mul
    if re.search(r"generator\.res\.\d+\.weight$", key) and ref.dim() == 2:
        return torch.eye(shape[0]) * math.sqrt(shape[0]) + 0.3 * r   # structure transform T_s (identity-ish)
    if ".norm" in key and key.endswith("style.weight"):
        return 0.5 * r / math.sqrt(shape[1])
    if ".norm" in key and key.endswith("style.bias"):
        half = shape[0] // 2
        out = 0.1 * r
        out[:half] += 1.0
        return out
    if key.endswith("to_rgb1.bias") or re.search(r"to_rgbs\.\d+\.bias$", key):
        return 0.05 * r
    if re.search(r"to_rgb(1|s\.\d+)\.conv\.weight$", key):
        return 0.35 * r                                          # keeps the image O(0.5)
    if ref.dim() == 5:
        return r                                                 # modulated conv weight [1,Cout,Cin,k,k]
    if re.search(r"res\.\d+\.conv2?\.0\.weight$", key):
        return 0.5 * r                                           # ModRes EqualConv2d (reference: randn*0.01)
    if ref.dim() == 4:
        fan_in = shape[1] * shape[2] * shape[3]
        if shape[0] <= 4:
            return r * math.sqrt(0.25 / fan_in)                  # 3-channel skip / mask heads
        return r * math.sqrt(1.9 / fan_in)                       # plain conv + LeakyReLU(0.2): variance-preserving
    if ref.dim() == 2:
        return r / math.sqrt(shape[1])
    if ref.dim() == 1:
        return 0.1 * r
    return r


def det_state_dict(template, seed: int = 0):
    """``template``: a state_dict (or module) giving keys and shapes -> deterministic fp32 CPU state_dict."""
    sd = template.state_dict() if hasattr(template, "state_dict") else template
    return {k: det_tensor(k, v, seed) for k, v in sd.items()}


def det_inputs(B: int, H: int, W: int, seed: int = 0, n_latent: int = 18):
    """Synthetic frame batch as the frame loop builds it (style_transfer.py:160-176): x = cat(RGB in [-1,1],
    parsing logits / 16), one W+ style code repeated over the batch."""
    g = torch.Generator(device="cpu")
    g.manual_seed(1234567 + seed)
    rgb = torch.rand((B, 3, H, W), generator=g) * 2 - 1
    parsing = torch.randn((B, 19, H, W), generator=g) / 16.0
    x = torch.cat([rgb, parsing], dim=1)
    style = torch.randn((1, n_latent, 512), generator=g).repeat(B, 1, 1)
    return x, style
