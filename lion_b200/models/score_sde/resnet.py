"""Global-latent prior -- mirror of the reference's models/score_sde/resnet.py
(Prior :124-218, ResBlockSEDrop :60-90, ResBlockSEClip :29-56, SE :16-27,
PriorSEDrop :221-224, PriorSEClip :226-229).  The forward is one C-ABI call
(`lion_global_prior_forward`, lion_b200/csrc/global_prior.cu).

When autograd needs it (grad mode on, and x requires grad, or the module is in train() mode and a parameter requires
grad) the forward is differentiable instead: the
training forward (`lion_global_prior_forward_train`) keeps the activations the backward reads, and the backward
(`lion_global_prior_backward`) gives the gradients of x and of every parameter.  In train() mode PriorSEDrop then
applies its dropout after each cell's first ReLU, with masks drawn on the device by torch.bernoulli_ (keep with
probability 1 - p, scaled by 1 / (1 - p), nn.Dropout's distribution); the random stream is not the one torch's fused
dropout kernel would draw."""
import ctypes as C
import functools

import torch
import torch.nn as nn

from ... import _lib as L


class SE(nn.Module):
    def __init__(self, channel, reduction=8):
        super().__init__()
        self.fc = nn.Sequential(nn.Conv2d(channel, channel // reduction, 1, 1, bias=False), nn.ReLU(inplace=True),
                                nn.Conv2d(channel // reduction, channel, 1, 1, bias=False), nn.Sigmoid())


class ResBlockSEClip(nn.Module):
    def __init__(self, input_dim, output_dim):
        super().__init__()
        self.input_dim, self.output_dim = input_dim, output_dim
        self.conv1 = nn.Conv2d(input_dim * 2, output_dim, 1, 1)
        self.conv2 = nn.Conv2d(output_dim, output_dim, 1, 1)
        self.SE = SE(output_dim)

    def __repr__(self):
        return "ResBlockSEClip(%d, %d)" % (self.input_dim, self.output_dim)


class ResBlockSEDrop(nn.Module):
    def __init__(self, input_dim, output_dim, dropout):
        super().__init__()
        self.input_dim, self.output_dim = input_dim, output_dim
        self.conv1 = nn.Conv2d(input_dim, output_dim, 1, 1)
        self.conv2 = nn.Conv2d(output_dim, output_dim, 1, 1)
        self.SE = SE(output_dim)
        self.dropout = nn.Dropout(dropout)
        self.dropout_ratio = dropout

    def __repr__(self):
        return "ResBlockSE_withdropout(%d, %d, drop=%f)" % (self.input_dim, self.output_dim, self.dropout_ratio)


class Prior(nn.Module):
    building_block = None

    def __init__(self, args, num_input_channels, *oargs, **kwargs):
        super().__init__()
        self.condition_input = kwargs.get('condition_input', False)
        self.cfg = oargs[0]
        self.clip_forge_enable = self.cfg.clipforge.enable
        self.num_scales = args.num_scales_dae
        self.num_input_channels = num_input_channels
        self.nf = nf = args.num_channels_dae
        if self.clip_forge_enable:
            self.clip_feat_mapping = nn.Conv1d(self.cfg.clipforge.feat_dim, self.nf, 1)
        self.mixed_prediction = args.mixed_prediction
        if self.mixed_prediction:
            raise NotImplementedError("lion_b200: sde.mixed_prediction is false in every shipped prior config")
        self.mixing_logit = None
        self.is_active = None
        self.embedding_dim = args.embedding_dim
        self.embedding_scale = args.embedding_scale
        assert args.embedding_type == 'positional', "lion_b200 implements the positional time embedding"
        self.temb_layer = nn.Sequential(nn.Conv2d(self.embedding_dim, self.embedding_dim * 4, 1, 1),
                                        nn.Conv2d(self.embedding_dim * 4, nf, 1, 1))
        self.input_layer = nn.Conv2d(num_input_channels, nf, 1, 1)
        self.all_modules = nn.ModuleList([self.building_block(nf, nf) for _ in range(args.num_cell_per_scale_dae)])
        self.output_layer = nn.Conv2d(nf, num_input_channels, 1, 1)

    def lion_desc(self):
        return [self.num_input_channels, self.nf, self.embedding_dim, len(self.all_modules), int(bool(self.clip_forge_enable)),
                self.cfg.clipforge.feat_dim, L.float_bits(self.embedding_scale)]

    def lion_params(self):
        ps = []
        if self.clip_forge_enable:
            ps += [self.clip_feat_mapping.weight, self.clip_feat_mapping.bias]
        ps += [self.temb_layer[0].weight, self.temb_layer[0].bias, self.temb_layer[1].weight, self.temb_layer[1].bias,
               self.input_layer.weight, self.input_layer.bias]
        for m in self.all_modules:
            ps += [m.conv1.weight, m.conv1.bias, m.conv2.weight, m.conv2.bias, m.SE.fc[0].weight, m.SE.fc[2].weight]
        return ps + [self.output_layer.weight, self.output_layer.bias]

    def forward(self, x, t, _drop_mask=None, **kwargs):
        """x [B, D, 1, 1], t [B] (or 0-dim) -> [B, D, 1, 1]   (resnet.py:195-218).  Differentiable in x and the
        parameters when grad mode is on and x requires grad, or the module is in train() mode and a parameter requires
        grad (the output is fp32, under autocast too); no gradient reaches t or clip_feat.  An eval() module called on
        an x that does not require grad returns a plain tensor, as sampling code calling it with grad mode on expects.
        _drop_mask [ncell, B, nf] fp32 (tests): the scaled dropout masks to apply in place of drawn ones."""
        params = self.lion_params()
        if torch.is_grad_enabled() and (x.requires_grad or (self.training and any(p.requires_grad for p in params))):
            return self._forward_train(x, t, params, _drop_mask, **kwargs)
        return self._forward_eval(x, t, **kwargs)

    def _time_clip(self, t, B, kwargs):
        t = t.detach().to(torch.float32)
        if t.dim() == 0:
            t = t.expand(1)
        if t.shape[0] == 1 and B > 1:
            t = t.expand(B)
        t = t.contiguous()
        clip = None
        if self.clip_forge_enable:
            clip = kwargs['clip_feat'].detach().to(torch.float32).contiguous()
        return t, clip

    @torch.no_grad()
    def _forward_eval(self, x, t, **kwargs):
        shape = x.shape
        B = shape[0]
        xin = x.detach().to(torch.float32).contiguous().view(B, -1)
        t, clip = self._time_clip(t, B, kwargs)
        m = L.model_for(self, L.KIND_GLOBAL_PRIOR, self.lion_desc(), self.lion_params())
        out = torch.empty_like(xin)
        with torch.cuda.device(xin.device):
            L.check(L.lib().lion_global_prior_forward(m.h, L.ptr(xin), L.ptr(t), L.ptr(clip), L.ptr(out), B, L.stream()),
                    "global_prior_forward")
        return out.view(shape)

    def _drop_masks(self, B, device):
        """Scaled dropout masks [ncell, B, nf] of ResBlockSEDrop in train() mode, or None (eval, p = 0, PriorSEClip)."""
        p = getattr(self.all_modules[0], 'dropout_ratio', 0.0) if self.training else 0.0
        if not p:
            return None
        keep = torch.empty(len(self.all_modules), B, self.nf, device=device).bernoulli_(1.0 - p)
        return keep.mul_(1.0 / (1.0 - p)) if p < 1.0 else keep

    def _forward_train(self, x, t, params, drop_mask, **kwargs):
        shape = x.shape
        B = shape[0]
        xin = x.to(torch.float32).contiguous().view(B, -1)
        t, clip = self._time_clip(t, B, kwargs)
        if drop_mask is None:
            drop_mask = self._drop_masks(B, xin.device)
        elif tuple(drop_mask.shape) != (len(self.all_modules), B, self.nf) or drop_mask.dtype != torch.float32:
            raise L.LionError("lion_b200: _drop_mask must be fp32 [%d, %d, %d], got %s %s"
                              % (len(self.all_modules), B, self.nf, drop_mask.dtype, tuple(drop_mask.shape)))
        else:
            drop_mask = drop_mask.detach().contiguous()
        m = L.model_for(self, L.KIND_GLOBAL_PRIOR, self.lion_desc(), params)
        return _PriorTrain.apply(m, t, clip, drop_mask, xin, *params).view(shape)


class _PriorTrain(torch.autograd.Function):
    """The global prior as one autograd node: inputs x [B, D] and the parameters in lion_params() order, one gradient
    for each.  Always fp32 (TF32 tensor cores), under autocast too, like the sampling forward."""

    @staticmethod
    @torch.amp.custom_fwd(device_type="cuda", cast_inputs=torch.float32)
    def forward(ctx, m, t, clip, drop_mask, x, *params):
        B = x.shape[0]
        lib = L.lib()
        saved = torch.empty(lib.lion_global_prior_saved_floats(m.h, B), device=x.device)
        out = torch.empty_like(x)
        with torch.cuda.device(x.device):
            L.check(lib.lion_global_prior_forward_train(m.h, L.ptr(x), L.ptr(t), L.ptr(clip), L.ptr(drop_mask),
                                                        L.ptr(saved), L.ptr(out), B, L.stream()),
                    "global_prior_forward_train")
        ctx.m = m
        ctx.save_for_backward(saved, clip, drop_mask, *params)    # params: autograd's check against in-place updates
        return out

    @staticmethod
    @torch.amp.custom_bwd(device_type="cuda")
    def backward(ctx, gout):
        if torch.is_grad_enabled():
            raise L.LionError("lion_b200: the global prior's backward is not itself differentiable "
                              "(double backward / create_graph=True is not supported)")
        saved, clip, drop_mask, *params = ctx.saved_tensors
        gout = gout.to(torch.float32).contiguous()
        B = gout.shape[0]
        gx = torch.empty_like(gout)
        gparams = [torch.empty_like(p) for p in params]
        arr = (C.c_void_p * len(gparams))(*[g.data_ptr() for g in gparams])
        with torch.cuda.device(gout.device):
            L.check(L.lib().lion_global_prior_backward(ctx.m.h, L.ptr(saved), L.ptr(clip), L.ptr(drop_mask), L.ptr(gout),
                                                       L.ptr(gx), arr, len(gparams), B, L.stream()),
                    "global_prior_backward")
        return (None, None, None, None, gx, *gparams)


class PriorSEDrop(Prior):
    def __init__(self, *args, **kwargs):
        self.building_block = functools.partial(ResBlockSEDrop, dropout=args[0].dropout)
        super().__init__(*args, **kwargs)


class PriorSEClip(Prior):
    building_block = ResBlockSEClip

    def __init__(self, *args, **kwargs):
        super().__init__(*args, **kwargs)
