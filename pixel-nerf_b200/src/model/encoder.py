"""Pixel-aligned image encoder (reference: src/model/encoder.py, SpatialEncoder).  The conv
trunk stays a library call (torchvision resnet + cuDNN): it runs once per scene and is a
"next" row of SURVEY.md section 8f, not part of the per-ray hot path.  `index()` here is
the torch/autograd version; inference gathers inside the fused kernels."""
import torch
import torch.nn.functional as F
import torchvision
from torch import nn

import pnr_native as pn
import util


class _UpsampleAC(torch.autograd.Function):
    """F.interpolate(x, size, mode="bilinear", align_corners=True) whose backward is pnr_upsample_bilinear_ac_backward,
    a gather in a fixed order: torch's CUDA backward adds with atomics and raises under
    torch.use_deterministic_algorithms(True).  The forward is torch's own call, so its output has the same bits."""

    @staticmethod
    def forward(ctx, x, size):
        ctx.in_hw = x.shape[-2:]
        ctx.dtype = x.dtype
        return F.interpolate(x, size, mode="bilinear", align_corners=True)

    @staticmethod
    def backward(ctx, d_out):
        return pn.upsample_bilinear_ac_backward(d_out, ctx.in_hw).to(ctx.dtype), None


class SpatialEncoder(nn.Module):
    def __init__(self, backbone="resnet34", pretrained=True, num_layers=4, index_interp="bilinear",
                 index_padding="border", upsample_interp="bilinear", feature_scale=1.0, use_first_pool=True,
                 norm_type="batch"):
        super().__init__()
        if backbone == "custom":
            raise NotImplementedError("encoder.backbone = custom (experimental ConvEncoder) is not provided")
        if index_interp != "bilinear" or index_padding != "border":
            raise NotImplementedError("only index_interp=bilinear / index_padding=border are supported")
        if norm_type != "batch":
            assert not pretrained
        self.feature_scale = feature_scale
        self.use_first_pool = use_first_pool
        self.num_layers = num_layers
        self.index_interp, self.index_padding, self.upsample_interp = index_interp, index_padding, upsample_interp
        print("Using torchvision", backbone, "encoder")
        self.model = getattr(torchvision.models, backbone)(
            weights="IMAGENET1K_V1" if pretrained else None, norm_layer=util.get_norm_layer(norm_type))
        self.model.fc = nn.Sequential()
        self.model.avgpool = nn.Sequential()
        self.latent_size = [0, 64, 128, 256, 512, 1024][num_layers]
        self.register_buffer("latent", torch.empty(1, 1, 1, 1), persistent=False)
        self.register_buffer("latent_scaling", torch.empty(2, dtype=torch.float32), persistent=False)

    def index(self, uv, cam_z=None, image_size=(), z_bounds=None):
        """uv (B,N,2) source-image pixels -> (B,L,N) bilinear, border-clamped (encoder.py:80-109)."""
        if uv.shape[0] == 1 and self.latent.shape[0] > 1:
            uv = uv.expand(self.latent.shape[0], -1, -1)
        if len(image_size) > 0:
            if len(image_size) == 1:
                image_size = (image_size, image_size)
            uv = uv * (self.latent_scaling / image_size) - 1.0
        out = F.grid_sample(self.latent, uv.unsqueeze(2), align_corners=True, mode=self.index_interp,
                            padding_mode=self.index_padding)
        return out[:, :, :, 0]

    def forward(self, x):
        """(B,3,H,W) -> latent (B,L,H/2,W/2): the four trunk maps, each bilinearly upsampled
        (align_corners=True) to the conv1 map's size, concatenated (encoder.py:111-164)."""
        if self.feature_scale != 1.0:
            up = self.feature_scale > 1.0
            x = F.interpolate(x, scale_factor=self.feature_scale, mode="bilinear" if up else "area",
                              align_corners=True if up else None, recompute_scale_factor=True)
        x = x.to(device=self.latent.device)
        m = self.model
        x = m.relu(m.bn1(m.conv1(x)))
        maps = [x]
        stages = [m.layer1, m.layer2, m.layer3, m.layer4][: self.num_layers - 1]
        for i, stage in enumerate(stages):
            if i == 0 and self.use_first_pool:
                x = m.maxpool(x)
            x = stage(x)
            maps.append(x)
        size = maps[0].shape[-2:]
        det = torch.are_deterministic_algorithms_enabled() and self.upsample_interp == "bilinear"
        maps = [_UpsampleAC.apply(t, size) if (det and t.is_cuda and t.requires_grad)
                else F.interpolate(t, size, mode=self.upsample_interp, align_corners=True) for t in maps]
        self.latents = maps
        self.latent = torch.cat(maps, dim=1)
        self.latent_scaling[0] = self.latent.shape[-1]
        self.latent_scaling[1] = self.latent.shape[-2]
        self.latent_scaling = self.latent_scaling / (self.latent_scaling - 1) * 2.0
        return self.latent

    @classmethod
    def from_conf(cls, conf):
        return cls(conf.get_string("backbone"), pretrained=conf.get_bool("pretrained", True),
                   num_layers=conf.get_int("num_layers", 4), index_interp=conf.get_string("index_interp", "bilinear"),
                   index_padding=conf.get_string("index_padding", "border"),
                   upsample_interp=conf.get_string("upsample_interp", "bilinear"),
                   feature_scale=conf.get_float("feature_scale", 1.0),
                   use_first_pool=conf.get_bool("use_first_pool", True))
