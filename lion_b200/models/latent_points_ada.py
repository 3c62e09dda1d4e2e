"""PVCNN2 U-Net and the VAE decoder built on it -- host-side mirror of the reference's
models/latent_points_ada.py (PVCNN2Unet :19-173, LatentPointDecPVC :222-272).

The whole U-Net forward is ONE C-ABI call (`lion_unet_forward`, lion_b200/csrc/net.cu): the
module tree below only owns the parameters (reference names, so checkpoints load unchanged)
and describes the architecture to the library.  `PointTransPVC` (the VAE *encoder*, :175-220)
runs on the same call with embed_dim = 0 and a 3-channel input.
"""
import torch
import torch.nn as nn

from .. import _lib as L
from .pvcnn2_ada import (create_pointnet2_sa_components, create_pointnet2_fp_modules, LinearAttention,
                         create_mlp_components, SharedMLP, PVConv, PointNetSAModule, PointNetFPModule)


def _blocks_of(layer):
    return list(layer) if isinstance(layer, nn.Sequential) else [layer]


class PVCNN2Unet(nn.Module):
    def __init__(self, num_classes, embed_dim, use_att, dropout=0.1, extra_feature_channels=3, input_dim=3,
                 width_multiplier=1, voxel_resolution_multiplier=1, time_emb_scales=1.0, verbose=True,
                 condition_input=False, point_as_feat=1, cfg={}, sa_blocks={}, fp_blocks={},
                 clip_forge_enable=0, clip_forge_dim=512):
        super().__init__()
        assert width_multiplier == 1 and voxel_resolution_multiplier == 1
        self.input_dim = input_dim
        self.clip_forge_enable = clip_forge_enable
        self.clip_forge_dim = clip_forge_dim
        self.sa_blocks = sa_blocks
        self.fp_blocks = fp_blocks
        self.point_as_feat = point_as_feat
        self.condition_input = condition_input
        assert extra_feature_channels >= 0
        self.extra_feature_channels = extra_feature_channels
        self.num_classes_out = num_classes
        self.use_att = use_att
        self.time_emb_scales = time_emb_scales
        self.embed_dim = embed_dim
        self.style_dim = cfg.latent_pts.style_dim
        if self.embed_dim > 0:
            self.embedf = nn.Sequential(nn.Linear(embed_dim, embed_dim), nn.LeakyReLU(0.1, inplace=True),
                                        nn.Linear(embed_dim, embed_dim))
        if self.clip_forge_enable:
            self.clip_forge_mapping = nn.Linear(clip_forge_dim, embed_dim)
            self.style_clip = nn.Linear(self.style_dim + embed_dim, self.style_dim)
        self.in_channels = extra_feature_channels + 3
        sa_layers, sa_in_channels, channels_sa_features, _ = create_pointnet2_sa_components(
            input_dim=input_dim, sa_blocks=self.sa_blocks, extra_feature_channels=extra_feature_channels,
            with_se=True, embed_dim=embed_dim, use_att=use_att, dropout=dropout, width_multiplier=width_multiplier,
            voxel_resolution_multiplier=voxel_resolution_multiplier, verbose=verbose, cfg=cfg)
        self.sa_layers = nn.ModuleList(sa_layers)
        self.global_att = None if not use_att else LinearAttention(channels_sa_features, 8, verbose=verbose)
        sa_in_channels[0] = extra_feature_channels + input_dim - 3
        fp_layers, channels_fp_features = create_pointnet2_fp_modules(
            fp_blocks=self.fp_blocks, in_channels=channels_sa_features, sa_in_channels=sa_in_channels, with_se=True,
            embed_dim=embed_dim, use_att=use_att, dropout=dropout, width_multiplier=width_multiplier,
            voxel_resolution_multiplier=voxel_resolution_multiplier, verbose=verbose, cfg=cfg)
        self.fp_layers = nn.ModuleList(fp_layers)
        layers, _ = create_mlp_components(in_channels=channels_fp_features, out_channels=[128, dropout, num_classes],
                                          classifier=True, dim=2, width_multiplier=width_multiplier, cfg=cfg)
        self.classifier = nn.ModuleList(layers)

    # ---- description of the network for the library (lion_b200/csrc/net.cu: build_unet) ----
    def lion_desc(self):
        d = [self.num_classes_out, self.embed_dim, self.extra_feature_channels, self.input_dim, int(bool(self.use_att)),
             int(bool(self.clip_forge_enable)), self.clip_forge_dim, self.style_dim, len(self.sa_blocks)]
        for conv_cfg, sa_cfg in self.sa_blocks:
            oc, nblk, res = conv_cfg if conv_cfg is not None else (0, 0, 0)
            m, radius, k, mlp = sa_cfg
            d += [int(conv_cfg is not None), oc, nblk, res, m, L.float_bits(radius), k, len(mlp)] + list(mlp)
        d.append(len(self.fp_blocks))
        for fp_cfg, conv_cfg in self.fp_blocks:
            oc, nblk, res = conv_cfg if conv_cfg is not None else (0, 0, 0)
            d += [len(fp_cfg)] + list(fp_cfg) + [int(conv_cfg is not None), oc, nblk, res]
        d.append(L.float_bits(self.time_emb_scales))       # sde.embedding_scale: t * scale enters the sinusoid
        return d

    def lion_params(self):
        ps = []
        if self.embed_dim > 0:
            ps += [self.embedf[0].weight, self.embedf[0].bias, self.embedf[2].weight, self.embedf[2].bias]
        if self.clip_forge_enable:
            ps += [self.clip_forge_mapping.weight, self.clip_forge_mapping.bias, self.style_clip.weight, self.style_clip.bias]
        for layer in self.sa_layers:
            for blk in _blocks_of(layer):
                ps += blk.lion_params()
        if self.global_att is not None:
            ps += self.global_att.lion_params()
        for layer in self.fp_layers:
            for blk in _blocks_of(layer):
                ps += blk.mlp.lion_params() if isinstance(blk, PointNetFPModule) else blk.lion_params()
        ps += self.classifier[0].lion_params() + [self.classifier[2].weight, self.classifier[2].bias]
        return ps

    @torch.no_grad()
    def forward_point_major(self, x, t=None, style=None, clip_feat=None, out=None):
        """x [B,N,D] (D = 3 + extra) fp32 -> [B,N,num_classes]; the layout the kernels use.

        Inside torch.autocast("cuda", dtype=torch.float16) the second 3x3x3 convolution of every PVConv takes FP16
        operands with fp32 accumulation (LION_FWD_CONV_FP16); everything else is computed as outside autocast, and the
        output stays fp32 where the reference's autocast route returns fp16 (a deviation in favour of precision)."""
        B, N, D = x.shape
        assert D == self.in_channels
        m = L.model_for(self, L.KIND_UNET, self.lion_desc(), self.lion_params())
        if out is None:
            out = torch.empty(B, N, self.num_classes_out, device=x.device, dtype=torch.float32)
        if self.embed_dim > 0:
            assert t is not None, 'require t'
            t = t.detach().to(torch.float32)
            if t.ndim == 0:
                t = t.view(1).expand(B)
            if t.ndim == 2 and t.shape[1] == 1:
                t = t[:, 0]
            t = t.contiguous()
        else:
            t = None
        if self.clip_forge_enable:
            assert clip_feat is not None, 'require clip_feat as input'
            clip_feat = clip_feat.detach().to(torch.float32).contiguous()
        else:
            clip_feat = None
        style = style.detach().to(torch.float32).contiguous()
        # The style (and clip_feat) is constant over the steps of a sampling run: everything that depends on it alone
        # (CLIP mixing, the 61 AdaGN Linears) is computed once per distinct style tensor.  The key is the storage
        # identity + version counter of the tensors; the cache holds a reference, so the storage cannot be recycled
        # for different values behind the key's back, and any in-place update bumps the version.
        key = (style.data_ptr(), style._version, tuple(style.shape),
               None if clip_feat is None else (clip_feat.data_ptr(), clip_feat._version), B)
        with torch.cuda.device(x.device):
            if getattr(m, "style_key", None) != key:
                L.check(L.lib().lion_unet_cache_style(m.h, L.ptr(style), L.ptr(clip_feat), B, L.stream()), "unet_cache_style")
                m.style_key, m.style_ref = key, (style, clip_feat)
            L.check(L.lib().lion_unet_forward_flags(m.h, L.ptr(x), L.ptr(t), None, None, L.ptr(out), B, N, L.forward_flags(),
                                                    L.stream()), "unet_forward")
        return out

    def forward(self, inputs, **kwargs):
        """inputs: [B, 3+extra, N] channel-major as in the reference (latent_points_ada.py:117-173)."""
        x = inputs.detach().to(torch.float32).permute(0, 2, 1).contiguous()
        out = self.forward_point_major(x, t=kwargs.get('t', None), style=kwargs['style'],
                                       clip_feat=kwargs.get('clip_feat', None))
        return out.permute(0, 2, 1).contiguous()


class PointTransPVC(nn.Module):
    """The VAE's latent-point encoder (reference: models/latent_points_ada.py:175-220): the same Ada U-Net with
    embed_dim = 0, no extra feature channel and 2*zdim + 2*input_dim outputs per point; x [B,N,3], style [B,S] ->
    {'mu_1d', 'sigma_1d'} [B, N*(input_dim + zdim)].  One lion_unet_forward call; the slicing below is the reference's."""
    sa_blocks = [
        ((32, 2, 32), (1024, 0.1, 32, (32, 64))),
        ((64, 3, 16), (256, 0.2, 32, (64, 128))),
        ((128, 3, 8), (64, 0.4, 32, (128, 256))),
        (None, (16, 0.8, 32, (128, 128, 128))),
    ]
    fp_blocks = [
        ((128, 128), (128, 3, 8)),
        ((128, 128), (128, 3, 8)),
        ((128, 128), (128, 2, 16)),
        ((128, 128, 64), (64, 2, 32)),
    ]

    def __init__(self, zdim, input_dim, args={}):
        super().__init__()
        assert zdim > 0
        self.zdim = zdim
        self.layers = PVCNN2Unet(2 * zdim + input_dim * 2, embed_dim=0, use_att=1, extra_feature_channels=0,
                                 input_dim=args.ddpm.input_dim, cfg=args, sa_blocks=self.sa_blocks, fp_blocks=self.fp_blocks,
                                 dropout=args.ddpm.dropout)
        self.skip_weight = args.latent_pts.skip_weight
        self.pts_sigma_offset = args.latent_pts.pts_sigma_offset
        self.input_dim = input_dim

    @torch.no_grad()
    def forward(self, inputs):
        x, style = inputs
        x = x.detach().to(torch.float32).contiguous()
        B, N, D = x.shape
        output = self.layers.forward_point_major(x, style=style)          # [B, N, 2*zdim + 2*input_dim]
        pt_mu_1d = self.skip_weight * output[:, :, :self.input_dim] + x
        pt_sigma_1d = output[:, :, self.input_dim:2 * self.input_dim] - self.pts_sigma_offset
        ft_mu_1d = output[:, :, 2 * self.input_dim:-self.zdim]
        ft_sigma_1d = output[:, :, -self.zdim:]
        mu_1d = torch.cat([pt_mu_1d, ft_mu_1d], dim=2).reshape(B, -1).contiguous()
        sigma_1d = torch.cat([pt_sigma_1d, ft_sigma_1d], dim=2).reshape(B, -1).contiguous()
        return {'mu_1d': mu_1d, 'sigma_1d': sigma_1d}


class LatentPointDecPVC(nn.Module):
    """input context: [B, Npoint*(3+D)] latent points; style [B, style_dim] -> points [B,N,3]"""
    sa_blocks = [
        ((32, 2, 32), (1024, 0.1, 32, (32, 64))),
        ((64, 3, 16), (256, 0.2, 32, (64, 128))),
        ((128, 3, 8), (64, 0.4, 32, (128, 256))),
        (None, (16, 0.8, 32, (128, 128, 128))),
    ]
    fp_blocks = [
        ((128, 128), (128, 3, 8)),
        ((128, 128), (128, 3, 8)),
        ((128, 128), (128, 2, 16)),
        ((128, 128, 64), (64, 2, 32)),
    ]

    def __init__(self, point_dim, context_dim, num_points=None, args={}, **kwargs):
        super().__init__()
        self.point_dim = point_dim
        self.context_dim = context_dim + self.point_dim
        self.num_points = args.data.tr_max_sample_points if num_points is None else num_points
        self.layers = PVCNN2Unet(point_dim, embed_dim=0, use_att=1, extra_feature_channels=context_dim,
                                 input_dim=args.ddpm.input_dim, cfg=args, sa_blocks=self.sa_blocks,
                                 fp_blocks=self.fp_blocks, dropout=args.ddpm.dropout)
        self.skip_weight = args.latent_pts.skip_weight

    @torch.no_grad()
    def forward(self, x, beta, context, style):
        assert context.shape[1] == self.num_points * self.context_dim
        context = context.detach().to(torch.float32).contiguous().view(-1, self.num_points, self.context_dim)
        xyz = context[:, :, :self.point_dim]
        output = self.layers.forward_point_major(context, style=style)
        return output * self.skip_weight + xyz
