"""PyTorch-CPU restatement of the reference model graph (test infrastructure).

Follows lib/models/resnet_video.py:133-351 (create_model), resnet_helper.py:35-194,
nonlocal_helper.py:29-213, head_helper.py:32-123, lfb_helper.py:43-338 and
model_builder_video.py:176-250 of the reference.  Every intermediate keeps the
reference blob name.  torch.autograd provides the backward oracle.

Parameters are a dict {reference_blob_name: tensor} in the reference's NCTHW
layouts (`{conv}_w` (Cout,Cin,kT,kH,kW), `{conv}_b`, `{x}_bn_s`, `{x}_bn_b`,
`pred_w` (classes,dim), `pred_b`).
"""
import math
from collections import OrderedDict

import torch
import torchvision.ops

from . import ops

BLOCK_CONFIG = {50: (3, 4, 6, 3), 101: (3, 4, 23, 3)}  # resnet_video.py:33-36


def obtain_arc(arc_type, video_length):
    """resnet_video.py:39-130 (only the I3D/C2D tables the shipped configs use)."""
    if arc_type == 1:
        tc = [[0], [0, 0, 0], [0, 0, 0, 0], [0] * 6, [0, 0, 0]]
    elif arc_type == 2:
        tc = [[2], [1, 1, 1], [1, 0, 1, 0], [1, 0, 1, 0, 1, 0], [0, 1, 0]]
    elif arc_type == 3:
        tc = [[0], [0, 0, 0], [0, 0, 0, 0], [0] * 23, [0, 0, 0]]
    elif arc_type == 4:
        tc = [[2], [1, 1, 1], [1, 0, 1, 0], [1 if i % 2 == 0 else 0 for i in range(23)], [0, 1, 0]]
    else:
        raise ValueError(arc_type)
    ts = [[1] * len(t) for t in tc]
    return tc, ts, int(video_length / 2)


class Graph(object):
    """Walks the reference graph; in 'spec' mode it only records parameter shapes,
    in 'run' mode it evaluates with torch ops."""

    def __init__(self, cfg, params=None, dropout_masks=None, emulate_tf32=False):
        """emulate_tf32: round (to nearest, straight-through gradient) every tensor that the tensor-core path
        stores as a TF32 tensor-core operand, at the same points of the graph (DESIGN.md section 3).  The
        resulting forward agrees with the GPU to fp32-accumulation error, so ReLU / max-pool decisions
        coincide and gradients can be compared tightly.  The default (False) is the plain fp32/fp64
        restatement of the reference."""
        self.emulate_tf32 = emulate_tf32
        self.cfg = cfg
        self.params = params
        self.spec = OrderedDict()       # name -> (shape, kind)
        self.blobs = OrderedDict()
        self.run = params is not None
        self.dilations = 1
        self.dropout_masks = dropout_masks or {}

    def q(self, x):
        if not self.emulate_tf32 or x is None:
            return x
        i = x.detach().to(torch.float32).contiguous().view(torch.int32)
        r = ((i + 0x1000) & ~0x1FFF).view(torch.float32).to(x.dtype)      # cvt.rna.tf32.f32
        return x + (r - x).detach()

    # ---- parameter helpers -------------------------------------------------
    def _p(self, name, shape, kind):
        self.spec[name] = (tuple(shape), kind)
        return self.params[name] if self.run else None

    def conv(self, x, name, cin, cout, kernels, strides=(1, 1, 1), pads=(0, 0, 0),
             dilations=(1, 1, 1), no_bias=1, kind='msra', round_out=True):
        w = self._p(name + '_w', (cout, cin) + tuple(kernels), kind)
        b = None if no_bias else self._p(name + '_b', (cout,), 'zero')
        if not self.run:
            return None
        y = ops.conv_nd(self.q(x), self.q(w), b, strides, pads, dilations)
        if round_out:
            y = self.q(y)
        self.blobs[name] = y
        return y

    def affine(self, x, name, dim):
        s = self._p(name + '_s', (dim,), 'affine_s')
        b = self._p(name + '_b', (dim,), 'affine_b')
        if not self.run:
            return None
        y = ops.affine_nd(x, s, b)
        self.blobs[name] = y
        return y

    def spatial_bn(self, x, name, dim, eps, momentum, gamma_kind='affine_s'):
        """model.SpatialBN (trainable BN): '_s' / '_b' trained, '_rm' / '_riv' running statistics; a training graph
        also yields '_sm' / '_siv' and the updated running statistics (recorded as '{name}_rm' / '{name}_riv')."""
        s = self._p(name + '_s', (dim,), gamma_kind)
        b = self._p(name + '_b', (dim,), 'affine_b')
        rm = self._p(name + '_rm', (dim,), 'bn_rm')
        rv = self._p(name + '_riv', (dim,), 'bn_riv')
        if not self.run:
            return None
        y, nrm, nrv, sm, siv = ops.spatial_bn(x, s, b, rm.detach(), rv.detach(), eps, momentum, self.test_mode)
        self.blobs[name] = y
        if not self.test_mode:
            self.blobs[name + '_rm'], self.blobs[name + '_riv'] = nrm, nrv
            self.blobs[name + '_sm'], self.blobs[name + '_siv'] = sm, siv
        return y

    def norm(self, x, name, dim):
        """AffineNd (MODEL.USE_AFFINE, every shipped config) or SpatialBN (resnet_helper.py / resnet_video.py:183-188)."""
        if self.cfg.MODEL.USE_AFFINE:
            return self.affine(x, name, dim)
        return self.spatial_bn(x, name, dim, self.cfg.MODEL.BN_EPSILON, self.cfg.MODEL.BN_MOMENTUM)

    def conv_affine(self, x, prefix, cin, cout, kernels, strides, pads, dilations=(1, 1, 1)):
        """ModelBuilder.Conv3dAffine (model_builder_video.py:200-221) / Conv3dBN (:176-197; it swallows `dilations` in
        **kwargs and never passes it to ConvNd, so a SpatialBN net only builds with MODEL.DILATIONS_AFTER_CONV5 False)."""
        if not self.cfg.MODEL.USE_AFFINE:
            dilations = (1, 1, 1)
        y = self.conv(x, prefix, cin, cout, kernels, strides, pads, dilations, no_bias=1, round_out=False)
        return self.norm(y, prefix + '_bn', cout)

    def relu(self, x):
        return self.q(torch.relu(x)) if self.run else None

    def dropout(self, x, name, ratio):
        """Caffe2 Dropout train mode: mask*x/(1-ratio).  Masks are injected (the
        Caffe2 RNG stream is unreproducible, SURVEY section 7)."""
        if not self.run:
            return None
        if name in self.dropout_masks:
            y = x * self.dropout_masks[name].to(x.dtype) / (1.0 - ratio)
        else:
            y = x  # parity runs: ratio treated as 0 unless a mask is injected
        self.blobs[name] = y
        return y

    # ---- resnet_helper.py --------------------------------------------------
    def bottleneck(self, x, dim_in, dim_out, stride, prefix, dim_inner, tc, ts):
        """bottleneck_transformation_3d (resnet_helper.py:35-72)."""
        d = self.dilations
        y = self.conv_affine(x, prefix + '_branch2a', dim_in, dim_inner, (1 + 2 * tc, 1, 1),
                             (ts, 1, 1), (tc, 0, 0))
        y = self.relu(y)
        y = self.conv_affine(y, prefix + '_branch2b', dim_inner, dim_inner, (1, 3, 3),
                             (1, stride, stride), (0, d, d), (1, d, d))
        y = self.relu(y)
        y = self.conv_affine(y, prefix + '_branch2c', dim_inner, dim_out, (1, 1, 1), (1, 1, 1), (0, 0, 0))
        return y

    def res_block(self, x, dim_in, dim_out, stride, prefix, dim_inner, tc, ts):
        """_generic_residual_block_3d + _add_shortcut_3d (resnet_helper.py:75-119)."""
        tr = self.bottleneck(x, dim_in, dim_out, stride, prefix, dim_inner, tc, ts)
        if dim_in == dim_out and ts == 1 and stride == 1:
            sc = x
        else:
            sc = self.conv_affine(x, prefix + '_branch1', dim_in, dim_out, (1, 1, 1), (ts, stride, stride), (0, 0, 0))
            if self.cfg.MODEL.USE_AFFINE:          # emulate_tf32: the fused conv + AffineNd epilogue stores it rounded
                sc = self.q(sc)
        if not self.run:
            return None
        y = self.q(torch.relu(tr + sc))
        self.blobs[prefix + '_branch2c_bn'] = y   # in-place Sum + Relu (resnet_helper.py:112-117)
        return y

    def res_stage(self, x, dim_in, dim_out, stride, num_blocks, prefix, dim_inner, tcs, tss,
                  batch_size=None, nonlocal_name=None, nonlocal_mod=1000, group=None):
        """res_stage_nonlocal / res_stage_nonlocal_group (resnet_helper.py:122-194).
        group = (pool_stride, spatial_dim, group_size) selects the grouped variant."""
        for idx in range(num_blocks):
            bstride = 2 if (idx == 0 and stride == 2) else 1
            x = self.res_block(x, dim_in, dim_out, bstride, '%s_%d' % (prefix, idx), dim_inner,
                               tcs[idx], tss[idx])
            dim_in = dim_out
            if idx % nonlocal_mod == nonlocal_mod - 1:
                name = '%s_%d' % (nonlocal_name, idx)
                if group is None:
                    x = self.add_nonlocal(x, dim_in, dim_in, batch_size, name, int(dim_in / 2))
                else:
                    x = self.add_nonlocal_group(x, dim_in, dim_in, batch_size, group[0], group[1],
                                                group[1], group[2], name, int(dim_in / 2))
        return x, dim_in

    # ---- nonlocal_helper.py ------------------------------------------------
    def spacetime_nonlocal(self, x, dim_in, dim_out, batch_size, prefix, dim_inner):
        """nonlocal_helper.py:29-160 (softmax + scale + maxpool + affine variant)."""
        nl = self.cfg.NONLOCAL
        nb = nl.NO_BIAS
        theta = self.conv(x, prefix + '_theta', dim_in, dim_inner, (1, 1, 1), no_bias=nb, kind='nl')
        if nl.USE_MAXPOOL:
            xp = ops.max_pool_nd(x, (1, 2, 2), (1, 2, 2), (0, 0, 0)) if self.run else None
            if self.run:
                self.blobs[prefix + '_pool'] = xp
        else:
            xp = x
        phi = self.conv(xp, prefix + '_phi', dim_in, dim_inner, (1, 1, 1), no_bias=nb, kind='nl')
        g = self.conv(xp, prefix + '_g', dim_in, dim_inner, (1, 1, 1), no_bias=nb, kind='nl')
        y = None
        if self.run:
            shape5d = theta.shape
            th = theta.reshape(batch_size, dim_inner, -1)
            ph = phi.reshape(batch_size, dim_inner, -1)
            gg = g.reshape(batch_size, dim_inner, -1)
            aff = self.q(ops.batch_matmul(th, ph, trans_a=1))         # (B, M, K)
            assert nl.USE_SOFTMAX, 'oracle covers the softmax variant used by every shipped config'
            if nl.USE_SCALE:
                aff = aff * (dim_inner ** -.5)
            self.blobs[prefix + '_affinity'] = aff
            p = self.q(ops.softmax_axis2(aff))
            self.blobs[prefix + '_affinity_prob'] = p
            t = self.q(ops.batch_matmul(gg, p, trans_b=1))            # (B, C/2, M)
            y = t.reshape(shape5d)
            self.blobs[prefix + '_y'] = y
        kind = 'zero_w' if nl.USE_ZERO_INIT_CONV else 'nl'
        out = self.conv(y, prefix + '_out', dim_inner, dim_out, (1, 1, 1), no_bias=nb, kind=kind,
                        round_out=not (nl.USE_AFFINE or nl.USE_BN))
        if nl.USE_BN:                                             # nonlocal_helper.py:146-155
            out = self.spatial_bn(out, prefix + '_bn', dim_out, nl.BN_EPSILON, nl.BN_MOMENTUM)
        if nl.USE_AFFINE:
            out = self.affine(out, prefix + '_bn', dim_out)
        return out

    def add_nonlocal(self, x, dim_in, dim_out, batch_size, prefix, dim_inner):
        """nonlocal_helper.py:163-171."""
        out = self.spacetime_nonlocal(x, dim_in, dim_out, batch_size, prefix, dim_inner)
        if not self.run:
            return None
        y = self.q(x + out)
        self.blobs[prefix + '_sum'] = y
        return y

    def add_nonlocal_group(self, x, dim_in, dim_out, batch_size, pool_stride, height, width,
                           group_size, prefix, dim_inner):
        """nonlocal_helper.py:174-213: groups of `group_size` consecutive frames."""
        group_num = int(pool_stride / group_size)
        assert pool_stride % group_size == 0
        if self.run and group_num > 1:
            x = x.permute(0, 2, 1, 3, 4)
            shape5d = x.shape
            x = x.reshape(batch_size * group_num, group_size, dim_in, height, width)
            x = x.permute(0, 2, 1, 3, 4)
        out = self.spacetime_nonlocal(x, dim_in, dim_out, batch_size * group_num, prefix, dim_inner)
        if not self.run:
            return None
        y = self.q(x + out)
        self.blobs[prefix + '_sum_grouped'] = y
        if group_num > 1:
            y = y.permute(0, 2, 1, 3, 4).reshape(shape5d).permute(0, 2, 1, 3, 4)
        self.blobs[prefix + '_sum'] = y
        return y

    # ---- lfb_helper.py -----------------------------------------------------
    def fbo_nl_head(self, box, dim_in, lfb, num_lfb_feat, test_mode, box_name='box_pooled'):
        """add_fbo_nl_head / prepare_nl_input / prepare_lfb / NLLayers / NLCore
        (lfb_helper.py:78-103, 160-338)."""
        cfg = self.cfg
        fb = cfg.FBO_NL
        nb = cfg.NONLOCAL.NO_BIAS
        d = fb.LATENT_DIM
        a, dim_a = box, dim_in
        if fb.INPUT_REDUCE_DIM:
            a = self.conv(a, box_name + '_fbonl_reduc', dim_in, d, (1, 1, 1), no_bias=nb, kind='fc')
            dim_a = d
        if fb.INPUT_DROPOUT_ON and not test_mode:
            a = self.dropout(a, (box_name + '_fbonl_reduc_fbonl_drop') if fb.INPUT_REDUCE_DIM
                             else (box_name + '_fbonl_drop'), fb.DROPOUT_RATE)
        b = None
        if self.run:
            # get_lfb_blob / NTC_to_NCT11 (lfb_helper.py:43-53,155-157)
            b = lfb.permute(0, 2, 1).reshape(-1, cfg.LFB.LFB_DIM, num_lfb_feat, 1, 1)
        b = self.conv(b, 'lfb_1x1', cfg.LFB.LFB_DIM, d, (1, 1, 1), no_bias=nb, kind='fc')
        if fb.LFB_DROPOUT_ON and not test_mode:
            b = self.dropout(b, 'lfb_1x1_drop', fb.DROPOUT_RATE)
        out = None
        for l in range(fb.NUM_LAYERS):
            pre = 'lfb_nl%d' % l
            theta = self.conv(a, pre + '_theta', dim_a, d, (1, 1, 1), no_bias=nb, kind='nl_default')
            phi = self.conv(b, pre + '_phi', d, d, (1, 1, 1), no_bias=nb, kind='nl_default')
            g = self.conv(b, pre + '_g', d, d, (1, 1, 1), no_bias=nb, kind='nl_default')
            t = None
            if self.run:
                th = theta.reshape(-1, d, 1)
                ph = phi.reshape(-1, d, num_lfb_feat)
                gg = g.reshape(-1, d, num_lfb_feat)
                aff = self.q(ops.batch_matmul(th, ph, trans_a=1))     # (R,1,L)
                if fb.SCALE:
                    aff = aff * (d ** -.5)
                self.blobs[pre + '_affinity'] = aff
                p = self.q(ops.softmax_axis2(aff))
                self.blobs[pre + '_affinity_prob'] = p
                t = self.q(ops.batch_matmul(gg, p, trans_b=1)).reshape(theta.shape)
                self.blobs[pre + '_y'] = t
                if fb.PRE_ACT:
                    if fb.PRE_ACT_LN:
                        t = ops.layer_norm_axis1(t)[0]
                        self.blobs[pre + '_y_ln'] = t
                    t = self.q(torch.relu(t))
            fused_sum = fb.PRE_ACT and not (fb.LFB_DROPOUT_ON and not test_mode)   # Conv -> Sum fused on the GPU
            o = self.conv(t, pre + '_out', d, dim_a, (1, 1, 1), no_bias=nb, kind='zero_w', round_out=not fused_sum)
            if not fb.PRE_ACT and self.run:
                o = ops.layer_norm_axis1(o)[0]
                self.blobs[pre + '_ln'] = o
            if fb.LFB_DROPOUT_ON and not test_mode:
                o = self.dropout(o, (pre + '_out_drop') if fb.PRE_ACT else (pre + '_ln_drop'),
                                 fb.DROPOUT_RATE)
            if self.run:
                out = self.q(o + a)
                self.blobs[pre + '_sum'] = out
                if not fb.PRE_ACT:
                    out = self.q(torch.relu(out))
                a = out
        return out, dim_a

    def fbo_pool_head(self, lfb, num_lfb_feat, kind):
        """add_fbo_avg_head / add_fbo_max_head (lfb_helper.py:106-127)."""
        if not self.run:
            return None, self.cfg.LFB.LFB_DIM
        b = lfb.permute(0, 2, 1).reshape(-1, self.cfg.LFB.LFB_DIM, num_lfb_feat, 1, 1)
        if kind == 'avg':
            y = ops.avg_pool_nd(b, (num_lfb_feat, 1, 1), (1, 1, 1), (0, 0, 0))
            self.blobs['fbo_avg_out'] = y
        else:
            y = ops.max_pool_nd(b, (num_lfb_feat, 1, 1), (1, 1, 1), (0, 0, 0))
            self.blobs['fbo_max_out'] = y
        return y, self.cfg.LFB.LFB_DIM

    def fbo_head(self, box, dim_in, lfb, num_lfb_feat, test_mode, box_name='box_pooled'):
        t = self.cfg.LFB.FBO_TYPE
        if t == 'nl':
            return self.fbo_nl_head(box, dim_in, lfb, num_lfb_feat, test_mode, box_name)
        return self.fbo_pool_head(lfb, num_lfb_feat, t)

    # ---- head_helper.py ----------------------------------------------------
    def roi_head(self, x, dim_in, proposals, lfb, lfb_infer_only, test_mode):
        """add_roi_head / roi_pool (head_helper.py:61-123)."""
        cfg = self.cfg
        box = None
        if self.run:
            pooled = ops.avg_pool_nd(x, (cfg.TRAIN.VIDEO_LENGTH // 2, 1, 1), (1, 1, 1), (0, 0, 0))
            self.blobs['blob_pooled'] = pooled
            p4 = pooled.squeeze(2)
            res = cfg.ROI.XFORM_RESOLUTION
            feat = torchvision.ops.roi_align(p4, proposals.to(p4.dtype), (res, res),
                                             spatial_scale=1.0 / cfg.ROI.SCALE_FACTOR,
                                             sampling_ratio=0, aligned=False)
            self.blobs['roi_feat_3d'] = feat
            if res > 1:
                feat = ops.max_pool_nd(feat, (res, res), (1, 1), (0, 0))
            box = feat.reshape(-1, dim_in, 1, 1, 1)
            self.blobs['box_pooled'] = box
        heads, dims = [box], [dim_in]
        if cfg.LFB.ENABLED and not lfb_infer_only:
            n = cfg.LFB.WINDOW_SIZE * cfg.AVA.LFB_MAX_NUM_FEAT_PER_STEP
            f, fd = self.fbo_head(box, dim_in, lfb, n, test_mode)
            heads.append(f)
            dims.append(fd)
        out = None
        if self.run:
            out = torch.cat(heads, dim=1)
            self.blobs['pool5'] = out
        return out, sum(dims)

    def basic_head(self, x, dim_in, pool_stride, out_spatial_dim, lfb, lfb_infer_only, test_mode):
        """add_basic_head (head_helper.py:32-58)."""
        cfg = self.cfg
        pooled = None
        if self.run:
            pooled = ops.avg_pool_nd(x, (pool_stride, out_spatial_dim, out_spatial_dim), (1, 1, 1), (0, 0, 0))
            self.blobs['res5_2_branch2c_bn_pooled'] = pooled
        heads, dims = [pooled], [dim_in]
        if cfg.LFB.ENABLED and not lfb_infer_only:
            f, fd = self.fbo_head(pooled, dim_in, lfb, cfg.LFB.WINDOW_SIZE, test_mode,
                                  box_name='res5_2_branch2c_bn_pooled')
            heads.append(f)
            dims.append(fd)
        out = None
        if self.run:
            out = torch.cat(heads, dim=1)
            self.blobs['pool5'] = out
        return out, sum(dims)

    # ---- resnet_video.py ---------------------------------------------------
    def create_model(self, inputs, split, lfb_infer_only=False):
        """resnet_video.create_model (resnet_video.py:133-351)."""
        cfg = self.cfg
        self.dilations = 1
        data = inputs.get('data') if self.run else None
        n1, n2, n3, n4 = BLOCK_CONFIG[cfg.MODEL.DEPTH]
        dim_inner = cfg.RESNETS.NUM_GROUPS * cfg.RESNETS.WIDTH_PER_GROUP
        test_mode = split in ('test', 'val')
        batch_size = int((cfg.TEST.BATCH_SIZE if test_mode else cfg.TRAIN.BATCH_SIZE) / cfg.NUM_GPUS)
        crop = cfg.TRAIN.CROP_SIZE if (split == 'train' and not lfb_infer_only) else cfg.TEST.CROP_SIZE
        if self.run:
            crop = data.shape[-1]
            batch_size = data.shape[0]
        tc, ts, pool_stride = obtain_arc(cfg.MODEL.VIDEO_ARC_CHOICE, cfg.TRAIN.VIDEO_LENGTH)
        self.test_mode = test_mode

        x = self.conv(data, 'conv1', 3, 64, (1 + tc[0][0] * 2, 7, 7), (ts[0][0], 2, 2), (tc[0][0], 3, 3),
                      round_out=False)
        x = self.norm(x, 'res_conv1_bn', 64)
        if self.run:
            x = self.q(torch.relu(x))
            self.blobs['res_conv1_bn'] = x
            x = ops.max_pool_nd(x, (1, 3, 3), (1, 2, 2), (0, 1, 1))
            self.blobs['pool1'] = x
        x, dim = self.res_stage(x, 64, 256, 1, n1, 'res2', dim_inner, tc[1], ts[1])
        layer_mod = cfg.NONLOCAL.LAYER_MOD
        if cfg.MODEL.DEPTH == 101:
            layer_mod = 2
        if not cfg.NONLOCAL.CONV3_NONLOCAL:
            layer_mod = 1000
        if self.run:
            x = ops.max_pool_nd(x, (2, 1, 1), (2, 1, 1), (0, 0, 0))
            self.blobs['pool2'] = x
        x, dim = self.res_stage(x, dim, 512, 2, n2, 'res3', dim_inner * 2, tc[2], ts[2],
                                batch_size=batch_size, nonlocal_name='nonlocal_conv3',
                                nonlocal_mod=layer_mod, group=(pool_stride, int(crop / 8), 4))
        layer_mod = cfg.NONLOCAL.LAYER_MOD
        if cfg.MODEL.DEPTH == 101:
            layer_mod = layer_mod * 4 - 1
        if not cfg.NONLOCAL.CONV4_NONLOCAL:
            layer_mod = 1000
        x, dim = self.res_stage(x, dim, 1024, 2, n3, 'res4', dim_inner * 4, tc[3], ts[3],
                                batch_size=batch_size, nonlocal_name='nonlocal_conv4',
                                nonlocal_mod=layer_mod)
        if cfg.MODEL.DILATIONS_AFTER_CONV5:
            self.dilations = 2
        x, dim = self.res_stage(x, dim, 2048, 1, n4, 'res5', dim_inner * 8, tc[4], ts[4])
        if self.run and cfg.MODEL.FREEZE_BACKBONE:
            x = x.detach()

        lfb = self.q(inputs.get('lfb')) if self.run else None     # the bank is fed TF32-rounded
        if cfg.DATASET == 'ava':
            out, dim = self.roi_head(x, dim, inputs.get('proposals') if self.run else None, lfb,
                                     lfb_infer_only, test_mode)
        else:
            out, dim = self.basic_head(x, dim, pool_stride, crop // 16, lfb, lfb_infer_only, test_mode)
        if lfb_infer_only:
            return None, None
        if cfg.TRAIN.DROPOUT_RATE > 0 and not test_mode:
            out = self.dropout(out, 'pool5_dropout', cfg.TRAIN.DROPOUT_RATE)
        w = self._p('pred_w', (cfg.MODEL.NUM_CLASSES, dim), 'fc')
        b = self._p('pred_b', (cfg.MODEL.NUM_CLASSES,), 'zero')
        if not self.run:
            return None, None
        pred = ops.fc(self.q(out), self.q(w), b)
        self.blobs['pred'] = pred
        scale = 1.0 / cfg.NUM_GPUS
        labels = inputs.get('labels')
        loss = None
        if cfg.MODEL.MULTI_LABEL:
            prob = torch.sigmoid(pred)
            if split == 'train':
                loss = ops.sigmoid_cross_entropy_loss(pred, labels, scale)
        else:
            if split == 'train':
                prob, loss = ops.softmax_with_loss(pred, labels, scale)
            else:
                prob = torch.softmax(pred, dim=1)
        self.blobs['prob'] = prob
        if loss is not None:
            self.blobs['loss'] = loss
        return prob, loss


def param_spec(cfg, split='train', lfb_infer_only=False):
    """OrderedDict name -> (shape, kind) of every parameter the graph creates."""
    g = Graph(cfg)
    g.create_model({}, split, lfb_infer_only)
    return g.spec


def make_params(cfg, seed=2, split='train', lfb_infer_only=False, dtype=torch.float32,
                nl_std=0.05, zero_init=False):
    """Deterministic synthetic parameters (SURVEY.md section 8d): MSRA conv weights, affine
    scale ~ U[0.5,1.5], bias ~ N(0,0.1); NL/FBO weights N(0,nl_std) and, unless
    zero_init, NON-zero `*_out_w` so that the NL / FBO branches contribute."""
    spec = param_spec(cfg, split, lfb_infer_only)
    gen = torch.Generator().manual_seed(seed)
    params = OrderedDict()
    for name, (shape, kind) in spec.items():
        if kind == 'msra':
            t = torch.randn(shape, generator=gen) * ops.msra_std(shape)
        elif kind == 'affine_s':
            t = torch.rand(shape, generator=gen) + 0.5
            if name.endswith('branch2c_bn_s') or name.startswith('nonlocal'):
                t = t * 0.25      # keep the residual stream O(1) through 16 blocks
        elif kind in ('affine_b', 'bn_rm'):
            t = torch.randn(shape, generator=gen) * 0.1
        elif kind == 'bn_riv':
            t = torch.rand(shape, generator=gen) + 0.5
        elif kind in ('nl', 'nl_default'):
            t = torch.randn(shape, generator=gen) * nl_std
        elif kind == 'zero_w':
            t = torch.zeros(shape) if zero_init else torch.randn(shape, generator=gen) * nl_std
        elif kind == 'fc':
            t = torch.randn(shape, generator=gen) * (cfg.MODEL.FC_INIT_STD if zero_init else 0.02)
        elif kind == 'zero':
            t = torch.zeros(shape) if zero_init else torch.randn(shape, generator=gen) * 0.05
        else:
            raise ValueError(kind)
        params[name] = t.to(dtype)
    return params


def make_inputs(cfg, n_clips=2, rois_per_clip=2, crop=None, frames=None, seed=0, lfb_len=None,
                dtype=torch.float32):
    """Synthetic inputs per SURVEY.md section 8d (configs 1/2)."""
    crop = crop or cfg.TRAIN.CROP_SIZE
    frames = frames or cfg.TRAIN.VIDEO_LENGTH
    g0 = torch.Generator().manual_seed(seed)
    inputs = {'data': torch.randn((n_clips, 3, frames, crop, crop), generator=g0).to(dtype)}
    if cfg.DATASET == 'ava':
        g1 = torch.Generator().manual_seed(seed + 1)
        r = n_clips * rois_per_clip
        idx = torch.arange(n_clips).repeat_interleave(rois_per_clip).to(torch.float32)
        half = crop / 2.0
        x1 = torch.rand(r, generator=g1) * (half - 1)
        y1 = torch.rand(r, generator=g1) * (half - 1)
        w = torch.rand(r, generator=g1) * (half - crop / 7.0) + crop / 7.0
        h = torch.rand(r, generator=g1) * (half - crop / 7.0) + crop / 7.0
        x2 = torch.clamp(x1 + w, max=crop - 1)
        y2 = torch.clamp(y1 + h, max=crop - 1)
        inputs['proposals'] = torch.stack([idx, x1, y1, x2, y2], dim=1).to(dtype)
        n_rows = r
    else:
        n_rows = n_clips
    g2 = torch.Generator().manual_seed(seed + 2)
    if cfg.MODEL.MULTI_LABEL:
        inputs['labels'] = (torch.rand((n_rows, cfg.MODEL.NUM_CLASSES), generator=g2) < 0.05).to(torch.int32)
    else:
        inputs['labels'] = torch.randint(0, cfg.MODEL.NUM_CLASSES, (n_rows,), generator=g2).to(torch.int32)
    if cfg.LFB.ENABLED:
        if lfb_len is None:
            lfb_len = (cfg.LFB.WINDOW_SIZE * cfg.AVA.LFB_MAX_NUM_FEAT_PER_STEP if cfg.DATASET == 'ava'
                       else cfg.LFB.WINDOW_SIZE)
        g3 = torch.Generator().manual_seed(seed + 3)
        lfb = torch.randn((n_rows, lfb_len, cfg.LFB.LFB_DIM), generator=g3) * 0.5
        lfb[:, lfb_len - int(math.ceil(lfb_len / 4.0)):, :] = 0.0   # zero padding rows (ava.py:310-321)
        inputs['lfb'] = lfb.to(dtype)
    return inputs


def forward(cfg, params, inputs, split='train', lfb_infer_only=False, dropout_masks=None, emulate_tf32=False):
    """Run the graph; returns (blobs OrderedDict, prob, loss)."""
    g = Graph(cfg, params, dropout_masks, emulate_tf32)
    prob, loss = g.create_model(inputs, split, lfb_infer_only)
    return g.blobs, prob, loss
