"""PVCNN2 building blocks with AdaGN -- host-side mirror of the reference's
models/pvcnn2_ada.py (same class names, constructor and forward signatures, and state_dict
keys, so released checkpoints load unchanged); every forward runs hand-written sm_90a
kernels through the C ABI of liblion_b200.so.  There is no PyTorch fallback.

  SE3d                      pvcnn2_ada.py:27-41     (parameters only; folded into PVConv's kernels)
  LinearAttention           pvcnn2_ada.py:43-71
  BallQuery                 pvcnn2_ada.py:86-118
  SharedMLP                 pvcnn2_ada.py:120-164
  Voxelization              pvcnn2_ada.py:166-193
  PVConv                    pvcnn2_ada.py:195-280
  PointNetSAModule          pvcnn2_ada.py:321-385
  PointNetFPModule          pvcnn2_ada.py:388-411
  create_mlp_components / create_pointnet2_sa_components / create_pointnet2_fp_modules  :416-567
"""
import functools

import torch
import torch.nn as nn

from ..third_party.pvcnn import functional as F
from .. import _lib as L
from .adagn import AdaGN


def _run(fn, *args):
    L.check(fn(*args), fn.__name__)


def _f32c(t):
    return t.detach().to(torch.float32).contiguous()


class Conv3d(nn.Conv3d):
    """nn.Conv3d(cin, cout, 3, stride=1, padding=1) as PVConv builds it (reference:
    models/pvcnn2_ada.py:211-222), evaluated stand-alone by the wgmma convolution kernel
    (lion_conv3d_gn_fwd).  Same parameters / state_dict keys as nn.Conv3d.  PVConv itself does
    not go through this class (its convolutions run inside the fused lion_pvconv_fwd /
    lion_unet_forward calls); it exists so the convolution can be used and checked on its own."""

    def __init__(self, in_channels, out_channels, kernel_size=3, stride=1, padding=1, bias=True):
        assert kernel_size == 3 and stride == 1 and padding == 1 and bias, \
            "lion_b200: only the 3x3x3 / stride 1 / padding 1 / bias convolution of PVConv is provided"
        super().__init__(in_channels, out_channels, 3, stride=1, padding=1, bias=True)

    def lion_params(self):
        return [self.weight, self.bias]

    @torch.no_grad()
    def forward(self, inputs, return_gn_stats=False):
        """inputs [B,Cin,r,r,r] -> [B,Cout,r,r,r]; with return_gn_stats also the per (shape, channel)
        sum and sum of squares over the voxels (float64 [B,Cout]) that the kernel's epilogue
        accumulates for the AdaGN that follows.

        Inside torch.autocast("cuda", dtype=torch.float16) the shapes of a PVConv's second convolution
        (Cin = Cout in {32, 64, 128}) run with FP16 operands (inputs and weights rounded to nearest even)
        and fp32 accumulation; other shapes run as outside autocast.  The output stays fp32 (the
        reference's cuDNN call returns fp16 there): a deviation in favour of precision."""
        B, C, r = inputs.shape[0], inputs.shape[1], inputs.shape[2]
        assert C == self.in_channels and inputs.dim() == 5 and inputs.shape[3] == r and inputs.shape[4] == r
        x = _f32c(inputs)
        m = L.model_for(self, L.KIND_CONV3D, [self.in_channels, self.out_channels, r], self.lion_params())
        out = torch.empty(B, self.out_channels, r, r, r, device=x.device, dtype=torch.float32)
        ssum = ssq = None
        if return_gn_stats:
            ssum = torch.empty(B, self.out_channels, device=x.device, dtype=torch.float64)
            ssq = torch.empty_like(ssum)
        with torch.cuda.device(x.device):
            _run(L.lib().lion_conv3d_gn_fwd_flags, m.h, L.ptr(x), L.ptr(out), L.ptr(ssum), L.ptr(ssq), B, L.forward_flags(),
                 L.stream())
        return (out, ssum, ssq) if return_gn_stats else out


class SE3d(nn.Module):
    def __init__(self, channel, reduction=8):
        super().__init__()
        self.fc = nn.Sequential(
            nn.Linear(channel, channel // reduction, bias=False), nn.ReLU(inplace=True),
            nn.Linear(channel // reduction, channel, bias=False), nn.Sigmoid())
        self.channel = channel

    def __repr__(self):
        return f"SE({self.channel}, {self.channel})"

    def lion_params(self):
        return [self.fc[0].weight, self.fc[2].weight]

    @torch.no_grad()
    def forward(self, inputs):
        """inputs [B,C,r,r,r] -> inputs * sigmoid(fc(mean_xyz inputs)) (stand-alone; PVConv folds this gate)."""
        shape = inputs.shape
        x = _f32c(inputs).view(shape[0], shape[1], -1)
        w1, w2 = self.fc[0].weight.detach().contiguous(), self.fc[2].weight.detach().contiguous()
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            _run(L.lib().lion_se3d_fwd, L.ctx(x.device), L.ptr(w1), L.ptr(w2), L.ptr(x), L.ptr(out), shape[0], shape[1],
                 x.shape[2], L.stream())
        return out.view(shape)


class LinearAttention(nn.Module):
    def __init__(self, dim, heads=4, dim_head=32, verbose=True):
        super().__init__()
        assert dim_head == 32, "lion_b200 kernels are specialised for dim_head == 32"
        self.heads = heads
        self.dim = dim
        hidden_dim = dim_head * heads
        self.to_qkv = nn.Conv2d(dim, hidden_dim * 3, 1, bias=False)
        self.to_out = nn.Conv2d(hidden_dim, dim, 1)

    def lion_params(self):
        return [self.to_qkv.weight, self.to_out.weight, self.to_out.bias]

    @torch.no_grad()
    def forward(self, x):
        """x: (B,C,N) -> (B,C,N)"""
        x = _f32c(x)
        B, C, N = x.shape
        m = L.model_for(self, L.KIND_ATTN, [self.dim, self.heads], self.lion_params())
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            _run(L.lib().lion_linear_attention_fwd, m.h, L.ptr(x), L.ptr(out), B, N, L.stream())
        return out


@torch.no_grad()
def swish(input):
    """x * sigmoid(x) (pvcnn2_ada.py:74-75); stand-alone kernel -- the fused blocks apply it on load."""
    x = _f32c(input)
    out = torch.empty_like(x)
    with torch.cuda.device(x.device):
        _run(L.lib().lion_swish_fwd, L.ptr(x), L.ptr(out), x.numel(), L.stream())
    return out


class Swish(nn.Module):
    """Keeps the reference's module numbering inside SharedMLP / PVConv; the fused blocks apply the
    activation inside their kernels, a stand-alone call runs `lion_swish_fwd`."""

    def forward(self, input):
        return swish(input)


class BallQuery(nn.Module):
    def __init__(self, radius, num_neighbors, include_coordinates=True):
        super().__init__()
        self.radius = radius
        self.num_neighbors = num_neighbors
        self.include_coordinates = include_coordinates

    @torch.no_grad()
    def forward(self, points_coords, centers_coords, points_features=None):
        points_coords = points_coords.contiguous()
        centers_coords = centers_coords.contiguous()
        neighbor_indices = F.ball_query(centers_coords, points_coords, self.radius, self.num_neighbors)
        neighbor_coordinates = F.grouping(points_coords, neighbor_indices)
        neighbor_coordinates = neighbor_coordinates - centers_coords.unsqueeze(-1)
        if points_features is None:
            assert self.include_coordinates, 'No Features For Grouping'
            return neighbor_coordinates
        neighbor_features = F.grouping(points_features, neighbor_indices)
        if self.include_coordinates:
            neighbor_features = torch.cat([neighbor_coordinates, neighbor_features], dim=1)
        return neighbor_features

    def extra_repr(self):
        return 'radius={}, num_neighbors={}{}'.format(
            self.radius, self.num_neighbors, ', include coordinates' if self.include_coordinates else '')


class SharedMLP(nn.Module):
    def __init__(self, in_channels, out_channels, dim=1, cfg={}):
        assert len(cfg) > 0, cfg
        super().__init__()
        conv = nn.Conv1d if dim == 1 else nn.Conv2d
        if not isinstance(out_channels, (list, tuple)):
            out_channels = [out_channels]
        self.in_channels = in_channels
        self.out_channels = list(out_channels)
        self.style_dim = cfg.latent_pts.style_dim
        layers = []
        for oc in out_channels:
            layers.append(conv(in_channels, oc, 1))
            layers.append(AdaGN(dim, cfg, oc))
            layers.append(Swish())
            in_channels = oc
        self.layers = nn.ModuleList(layers)

    def lion_params(self):
        ps = []
        for l in self.layers:
            if isinstance(l, AdaGN):
                ps += l.lion_params()
            elif not isinstance(l, Swish):
                ps += [l.weight, l.bias]
        return ps

    @torch.no_grad()
    def _run(self, x, style):
        shape = x.shape
        x = _f32c(x).reshape(shape[0], shape[1], -1)
        style = _f32c(style)
        B, C, R = x.shape
        m = L.model_for(self, L.KIND_SHARED_MLP,
                        [self.in_channels, self.style_dim, len(self.out_channels)] + self.out_channels,
                        self.lion_params())
        out = torch.empty(B, self.out_channels[-1], R, device=x.device, dtype=torch.float32)
        with torch.cuda.device(x.device):
            _run(L.lib().lion_shared_mlp_fwd, m.h, L.ptr(x), L.ptr(style), L.ptr(out), B, R, L.stream())
        return out.reshape(B, self.out_channels[-1], *shape[2:])

    def forward(self, *inputs):
        if len(inputs) == 1 and len(inputs[0]) == 4:
            inputs = inputs[0]
        if len(inputs) == 4:
            x, _, _, style = inputs
            return (self._run(x, style), *inputs[1:])
        elif len(inputs) == 2:
            x, style = inputs
            return self._run(x, style)
        raise NotImplementedError


class Voxelization(nn.Module):
    def __init__(self, resolution, normalize=True, eps=0):
        super().__init__()
        self.r = int(resolution)
        self.normalize = normalize
        self.eps = eps

    @torch.no_grad()
    def forward(self, features, coords):
        norm_coords, vox_coords = F.voxel_coords(coords.detach(), self.r, self.normalize, self.eps)
        if features is None:
            return features, norm_coords
        return F.avg_voxelize(features, vox_coords, self.r), norm_coords

    def extra_repr(self):
        return 'resolution={}{}'.format(self.r, ', normalized eps = {}'.format(self.eps) if self.normalize else '')


class PVConv(nn.Module):
    def __init__(self, in_channels, out_channels, kernel_size, resolution, normalize=1, eps=0, with_se=False,
                 add_point_feat=True, attention=False, dropout=0.1, verbose=True, cfg={}):
        super().__init__()
        assert len(cfg) > 0, cfg
        assert kernel_size == 3 and with_se and add_point_feat and normalize and eps == 0, \
            "lion_b200 implements the PVConv variant LION instantiates (3x3x3, SE, point branch, normalised coords)"
        self.in_channels, self.out_channels = in_channels, out_channels
        self.resolution = resolution
        self.style_dim = cfg.latent_pts.style_dim
        self.voxelization = Voxelization(resolution, normalize=normalize, eps=eps)
        NormLayer = functools.partial(AdaGN, 3, cfg)
        voxel_layers = [
            nn.Conv3d(in_channels, out_channels, kernel_size, stride=1, padding=kernel_size // 2),
            NormLayer(out_channels), Swish(), nn.Dropout(dropout),
            nn.Conv3d(out_channels, out_channels, kernel_size, stride=1, padding=kernel_size // 2),
            NormLayer(out_channels)]
        if with_se:
            voxel_layers.append(SE3d(out_channels))
        self.voxel_layers = nn.ModuleList(voxel_layers)
        self.attn = LinearAttention(out_channels, verbose=verbose) if attention else None
        if add_point_feat:
            self.point_features = SharedMLP(in_channels, out_channels, cfg=cfg)
        self.add_point_feat = add_point_feat

    def lion_desc(self):
        return [self.in_channels, self.out_channels, self.resolution, int(self.attn is not None), self.style_dim]

    def lion_params(self):
        v = self.voxel_layers
        ps = [v[0].weight, v[0].bias] + v[1].lion_params() + [v[4].weight, v[4].bias] + v[5].lion_params() + v[6].lion_params()
        if self.attn is not None:
            ps += self.attn.lion_params()
        return ps + self.point_features.lion_params()

    @torch.no_grad()
    def forward(self, inputs):
        features, coords_input, time_emb, style = inputs[0], inputs[1], inputs[2], inputs[3]
        coords = coords_input[:, :3] if coords_input.shape[1] > 3 else coords_input
        assert features.shape[0] == coords.shape[0] and features.shape[2] == coords.shape[2], \
            f'get feat: {features.shape} and {coords.shape}'
        assert coords.shape[1] == 3, f'expect coords: B,3,Npoint, get: {coords.shape}'
        features, coords, style = _f32c(features), _f32c(coords), _f32c(style)
        B, _, N = features.shape
        m = L.model_for(self, L.KIND_PVCONV, self.lion_desc(), self.lion_params())
        out = torch.empty(B, self.out_channels, N, device=features.device, dtype=torch.float32)
        with torch.cuda.device(features.device):
            _run(L.lib().lion_pvconv_fwd, m.h, L.ptr(features), L.ptr(coords), L.ptr(style), L.ptr(out), B, N, L.stream())
        return out, coords_input, time_emb, style


class PointNetSAModule(nn.Module):
    def __init__(self, num_centers, radius, num_neighbors, in_channels, out_channels, include_coordinates=True, cfg={}):
        super().__init__()
        assert include_coordinates and not isinstance(radius, (list, tuple)), \
            "lion_b200 implements the single-scale SA module LION instantiates"
        out_channels = list(out_channels) if isinstance(out_channels, (list, tuple)) else [out_channels]
        self.num_centers, self.radius, self.num_neighbors = num_centers, radius, num_neighbors
        self.in_channels = in_channels
        self.style_dim = cfg.latent_pts.style_dim
        self.out_channels = out_channels[-1]
        self.groupers = nn.ModuleList([BallQuery(radius=radius, num_neighbors=num_neighbors, include_coordinates=True)])
        self.mlps = nn.ModuleList([SharedMLP(in_channels=in_channels + 3, out_channels=out_channels, dim=2, cfg=cfg)])

    def lion_desc(self):
        oc = self.mlps[0].out_channels
        return [self.in_channels, self.num_centers, L.float_bits(self.radius), self.num_neighbors, self.style_dim, len(oc)] + oc

    def lion_params(self):
        return self.mlps[0].lion_params()

    @torch.no_grad()
    def forward(self, inputs):
        features, coords, time_emb, style = inputs[0], inputs[1], inputs[2], inputs[3]
        if coords.shape[1] > 3:
            coords = coords[:, :3]
        features, coords, style = _f32c(features), _f32c(coords), _f32c(style)
        B, _, N = features.shape
        M = self.num_centers
        m = L.model_for(self, L.KIND_SA, self.lion_desc(), self.lion_params())
        out = torch.empty(B, self.out_channels, M, device=features.device, dtype=torch.float32)
        centers = torch.empty(B, 3, M, device=features.device, dtype=torch.float32)
        with torch.cuda.device(features.device):
            _run(L.lib().lion_sa_module_fwd, m.h, L.ptr(features), L.ptr(coords), L.ptr(style), L.ptr(out), L.ptr(centers),
                 B, N, L.stream())
        if time_emb is not None and type(time_emb) is not dict:
            time_emb = time_emb[:, :, :M]
        return out, centers, time_emb, style

    def extra_repr(self):
        return f'num_centers={self.num_centers}, out_channels={self.out_channels}'


class PointNetFPModule(nn.Module):
    def __init__(self, in_channels, out_channels, cfg={}):
        super().__init__()
        self.mlp = SharedMLP(in_channels=in_channels, out_channels=out_channels, dim=1, cfg=cfg)
        self.in_channels = in_channels
        self.style_dim = cfg.latent_pts.style_dim

    @torch.no_grad()
    def forward(self, inputs):
        if len(inputs) == 5:
            points_coords, centers_coords, centers_features, time_emb, style = inputs
            points_features = None
        elif len(inputs) == 6:
            points_coords, centers_coords, centers_features, points_features, time_emb, style = inputs
        else:
            raise NotImplementedError
        pc, cc, cf, style = _f32c(points_coords[:, :3]), _f32c(centers_coords[:, :3]), _f32c(centers_features), _f32c(style)
        pf = _f32c(points_features) if points_features is not None else None
        B, Cc, M = cf.shape
        N = pc.shape[2]
        Cp = pf.shape[1] if pf is not None else 0
        assert Cc + Cp == self.in_channels, f'expect {self.in_channels} input channels, get {Cc}+{Cp}'
        oc = self.mlp.out_channels
        # the packed model depends on the (interpolated | skip) split, which is a call-time property
        key = (Cc, Cp)
        if self.__dict__.get("_lion_split") != key:
            self.__dict__["_lion_split"] = key
            self.__dict__.pop("_lion_model", None)
        m = L.model_for(self, L.KIND_FP, [Cc, Cp, self.style_dim, len(oc)] + oc, self.mlp.lion_params())
        out = torch.empty(B, oc[-1], N, device=cf.device, dtype=torch.float32)
        with torch.cuda.device(cf.device):
            _run(L.lib().lion_fp_module_fwd, m.h, L.ptr(pc), L.ptr(cc), L.ptr(cf), L.ptr(pf), L.ptr(style), L.ptr(out),
                 B, N, M, L.stream())
        if time_emb is not None:
            time_emb = time_emb[:, :, 0:1].expand(-1, -1, N)
        return out, points_coords, time_emb, style


def create_mlp_components(in_channels, out_channels, classifier=False, dim=2, width_multiplier=1, cfg={}):
    """reference: pvcnn2_ada.py:416-446 (dim=2, classifier=True is the only form LION uses)."""
    assert dim == 2 and classifier, "lion_b200 builds the classifier head form only"
    r = width_multiplier
    layers = []
    for oc in out_channels[:-1]:
        if oc < 1:
            layers.append(nn.Dropout(oc))
        else:
            oc = int(r * oc)
            layers.append(SharedMLP(in_channels, oc, cfg=cfg))
            in_channels = oc
    layers.append(nn.Conv1d(in_channels, out_channels[-1], 1))
    return layers, out_channels[-1]


def create_pointnet2_sa_components(sa_blocks, extra_feature_channels, input_dim=3, embed_dim=64, use_att=False,
                                   force_att=0, dropout=0.1, with_se=False, normalize=True, eps=0, has_temb=1,
                                   width_multiplier=1, voxel_resolution_multiplier=1, verbose=True, cfg={}):
    """reference: pvcnn2_ada.py:448-517.  Keeps its module-table quirk: levels > 0 register only
    their first PVConv (`if c == 0 ... elif k == 0`, :484-489) -- it defines the checkpoint layout."""
    assert len(cfg) > 0, cfg
    r, vr = width_multiplier, voxel_resolution_multiplier
    in_channels = extra_feature_channels + input_dim
    sa_layers, sa_in_channels = [], []
    num_centers = None
    for c, (conv_configs, sa_configs) in enumerate(sa_blocks):
        k = 0
        sa_in_channels.append(in_channels)
        blocks = []
        if conv_configs is not None:
            out_channels, num_blocks, voxel_resolution = conv_configs
            out_channels = int(r * out_channels)
            for p in range(num_blocks):
                attention = ((c + 1) % 2 == 0 and use_att and p == 0) or (force_att and c > 0)
                block = functools.partial(PVConv, kernel_size=3, resolution=int(vr * voxel_resolution),
                                          attention=attention, dropout=dropout, with_se=with_se,
                                          normalize=normalize, eps=eps, verbose=verbose, cfg=cfg)
                if c == 0:
                    blocks.append(block(in_channels, out_channels))
                elif k == 0:
                    blocks.append(block(in_channels + embed_dim * has_temb, out_channels))
                in_channels = out_channels
                k += 1
            extra_feature_channels = in_channels
        if sa_configs is not None:
            num_centers, radius, num_neighbors, out_channels = sa_configs
            out_channels = [int(r * oc) for oc in out_channels]
            blocks.append(PointNetSAModule(cfg=cfg, num_centers=num_centers, radius=radius, num_neighbors=num_neighbors,
                                           in_channels=extra_feature_channels + (embed_dim * has_temb if k == 0 else 0),
                                           out_channels=out_channels, include_coordinates=True))
            in_channels = extra_feature_channels = blocks[-1].out_channels
        sa_layers.append(blocks[0] if len(blocks) == 1 else nn.Sequential(*blocks))
    return sa_layers, sa_in_channels, in_channels, 1 if num_centers is None else num_centers


def create_pointnet2_fp_modules(fp_blocks, in_channels, sa_in_channels, embed_dim=64, use_att=False, dropout=0.1,
                                has_temb=1, with_se=False, normalize=True, eps=0, width_multiplier=1,
                                voxel_resolution_multiplier=1, verbose=True, cfg={}):
    """reference: pvcnn2_ada.py:520-567.  No FP PVConv ever gets attention there (its predicate
    compares against a shadowed, one-element list, :531-546); reproduced by construction."""
    assert len(cfg) > 0, cfg
    r, vr = width_multiplier, voxel_resolution_multiplier
    fp_layers = []
    for fp_idx, (fp_configs, conv_configs) in enumerate(fp_blocks):
        blocks = []
        out_channels = tuple(int(r * oc) for oc in fp_configs)
        blocks.append(PointNetFPModule(in_channels=in_channels + sa_in_channels[-1 - fp_idx] + embed_dim * has_temb,
                                       out_channels=out_channels, cfg=cfg))
        in_channels = out_channels[-1]
        if conv_configs is not None:
            out_channels, num_blocks, voxel_resolution = conv_configs
            out_channels = int(r * out_channels)
            for p in range(num_blocks):
                blocks.append(PVConv(in_channels, out_channels, kernel_size=3, resolution=int(vr * voxel_resolution),
                                     attention=False, dropout=dropout, with_se=with_se, normalize=normalize, eps=eps,
                                     verbose=verbose, cfg=cfg))
                in_channels = out_channels
        fp_layers.append(blocks[0] if len(blocks) == 1 else nn.Sequential(*blocks))
    return fp_layers, in_channels
