"""Seeded VGG19 features and inputs for the VGG loss tests (no pretrained weights: they cannot be downloaded)."""
import torch

SEED = 2019


def seeded_features(seed=SEED):
    """torchvision's vgg19().features layout with He-normal filters and N(0, 1) biases drawn from ``seed`` (deterministic on the
    CPU)."""
    from torchvision.models import vgg
    features = vgg.make_layers(vgg.cfgs['E'])
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for m in features:
            if isinstance(m, torch.nn.Conv2d):
                fan_in = m.in_channels * 9
                m.weight.copy_(torch.randn(m.weight.shape, generator=g) * (2.0 / fan_in) ** 0.5)
                m.bias.copy_(torch.randn(m.bias.shape, generator=g))
    return features


def seeded_images(B, H, W, seed):
    """Two [B, 3, H, W] f32 images in [0, 1)."""
    g = torch.Generator().manual_seed(seed)
    return torch.rand((B, 3, H, W), generator=g), torch.rand((B, 3, H, W), generator=g)
