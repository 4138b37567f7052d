"""CNNModelHelper stand-in: the op-emitter object the reference's builders call
(`model.ConvNd`, `model.MaxPool`, `model.net.Sum`, ... -- the list is in SURVEY.md
section 8b).  Emitters only RECORD ops and parameter initialisers; the executor
(vlfb/executor.py) lowers the recorded net onto the sm_90a kernels.

Argument conventions follow the Caffe2 python helpers at the reference's call sites
(e.g. lib/models/resnet_video.py:169-179 for ConvNd, :190-196 for MaxPool).
"""
from .net import Net, _as_list


class CNNModelHelper(object):
    def __init__(self, order='NCHW', name=None, use_cudnn=True, cudnn_exhaustive_search=False,
                 ws_nbytes_limit=None, init_params=True, use_mem_cache=False, **kwargs):
        assert order == 'NCHW', 'the reference only builds NCHW nets (model_builder_video.py:69)'
        self.name = name or 'model'
        self.order = order
        self.use_cudnn = use_cudnn                      # accepted, meaningless here
        self.cudnn_exhaustive_search = cudnn_exhaustive_search
        self.ws_nbytes_limit = ws_nbytes_limit
        self.init_params = init_params
        self.net = Net(self.name)
        self.param_init_net = Net(self.name + '_init')
        self.net._model = self
        self.param_init_net._model = self
        self.params = []
        self.weights = []
        self.biases = []
        self.param_to_grad = {}
        self.frozen_params = set()                      # AffineNd scale/bias, SpatialBN running statistics: no gradient op
        self.computed_params = []                       # SpatialBN '_rm' / '_riv' (Caffe2: computed params)
        self._owner = None                              # CompiledNet once created

    # ---- parameters ------------------------------------------------------------
    def GetParams(self, namescope=None):
        return list(self.params)

    def GetComputedParams(self, namescope=None):
        return list(self.computed_params)       # SpatialBN running statistics ('_rm', '_riv'); none in the Affine variant

    def GetAllParams(self, namescope=None):
        return self.GetParams(namescope) + self.GetComputedParams(namescope)

    def _make_param(self, name, shape, init, is_weight):
        init_type, init_args = init
        getattr(self.param_init_net, init_type)([], name, shape=list(shape), **init_args)
        if name not in self.params:
            self.params.append(name)
            (self.weights if is_weight else self.biases).append(name)
            self.net.Proto().external_input.append(name)
        return name

    # ---- layers with parameters ------------------------------------------------
    def ConvNd(self, blob_in, blob_out, dim_in, dim_out, kernel, weight_init=None, bias_init=None,
               strides=None, pads=None, no_bias=0, group=1, dilations=None, **kwargs):
        kernels = list(kernel) if isinstance(kernel, (list, tuple)) else [kernel] * 3
        group = int(group)
        if group > 1:
            # Caffe2 grouped Conv (ResNeXt branch2b, resnet_helper.py bottleneck_transformation_3d): the CUDA-core
            # kernels of csrc/gconv.cu take per-group widths that are multiples of 4 in [4, 64], spatial kernels only
            cig, cog = dim_in // group, dim_out // group
            if dim_in % group or dim_out % group or not all(c % 4 == 0 and 4 <= c <= 64 for c in (cig, cog)):
                raise ValueError('%s: grouped conv %d -> %d channels in %d groups needs per-group widths that are '
                                 'multiples of 4 in [4, 64]' % (blob_out, dim_in, dim_out, group))
            if len(kernels) != 3 or kernels == [1, 1, 1]:
                raise ValueError('%s: grouped convs need a 3-D spatial kernel (no grouped 1x1x1 conv)' % blob_out)
        elif group != 1:
            raise ValueError('%s: group must be >= 1, got %d' % (blob_out, group))
        w = self._make_param(blob_out + '_w', [dim_out, dim_in // group] + kernels,
                             weight_init or ('XavierFill', {}), True)
        inputs = [blob_in, w]
        if not no_bias:
            inputs.append(self._make_param(blob_out + '_b', [dim_out],
                                           bias_init or ('ConstantFill', {'value': 0.}), False))
        extra = {'group': group} if group > 1 else {}
        return self.net.Conv(inputs, blob_out, kernels=kernels,
                             strides=list(strides or [1] * len(kernels)),
                             pads=list(pads or [0] * (2 * len(kernels))),
                             dilations=list(dilations or [1] * len(kernels)), order=self.order, **extra)

    def FC(self, blob_in, blob_out, dim_in, dim_out, weight_init=None, bias_init=None, **kwargs):
        w = self._make_param(blob_out + '_w', [dim_out, dim_in], weight_init or ('XavierFill', {}), True)
        b = self._make_param(blob_out + '_b', [dim_out], bias_init or ('ConstantFill', {'value': 0.}), False)
        return self.net.FC([blob_in, w, b], blob_out)

    def SpatialBN(self, blob_in, blob_out, dim_in, epsilon=1e-5, momentum=0.9, is_test=False, **kwargs):
        """Trainable batch normalisation as the reference emits it (model_builder_video.py:186-190,
        resnet_video.py:185-188, nonlocal_helper.py:146-150): parameters '{out}_s' (1) / '{out}_b' (0) are trained,
        '{out}_rm' (0) / '{out}_riv' (1; a running VARIANCE, lib/utils/bn_helper.py:216-219) are computed parameters.
        Training nets also emit '{out}_sm' / '{out}_siv' (batch mean / inverse std), which precise-BN reads
        (bn_helper.py:170-173).  Statistics are per process (= per GPU), as in the reference."""
        scale = self._make_param(blob_out + '_s', [dim_in], ('ConstantFill', {'value': 1.}), True)
        bias = self._make_param(blob_out + '_b', [dim_in], ('ConstantFill', {'value': 0.}), False)
        stats = []
        for sfx, val in (('_rm', 0.), ('_riv', 1.)):
            name = blob_out + sfx
            self.param_init_net.ConstantFill([], name, shape=[dim_in], value=val)
            if name not in self.computed_params:
                self.computed_params.append(name)
                self.net.Proto().external_input.append(name)
            self.frozen_params.add(name)
            stats.append(name)
        outs = [blob_out] if is_test else [blob_out, stats[0], stats[1], blob_out + '_sm', blob_out + '_siv']
        res = self.net.SpatialBN([blob_in, scale, bias] + stats, outs, epsilon=float(epsilon), momentum=float(momentum),
                                 is_test=bool(is_test), order=self.order)
        return res[0] if isinstance(res, (list, tuple)) else res

    def FboNLStack(self, blob_a, blob_b, prefix, dim_a, dim_b, latent_dim, num_feat2, num_layers, init1, init2,
                   scale=1.0, pre_act_ln=True, dropout_ratio=0.0):
        """All layers of lfb_helper.NLLayers (one query per RoI, FBO_NL.PRE_ACT) as ONE operator (B200.FBO_STACK).
        Creates exactly the parameters NLCore's four ConvNd calls create -- '{prefix}_nl{l}_{theta,phi,g,out}_w/_b'
        with their 5-D conv shapes and initialisers -- so checkpoints are interchangeable with the as-written graph,
        and emits the blobs '{prefix}_nl{l}_{theta,affinity_prob,y,out,sum}'; phi / g / affinity are never formed
        (vlfb_fbo_nl_fwd, csrc/fbo.cu section 3).  Returns the last layer's sum."""
        inputs, outputs = [blob_a, blob_b], []
        for layer in range(num_layers):
            name = prefix + '_nl%d' % layer
            for part, (dout, din, init) in (('theta', (latent_dim, dim_a, init1)), ('phi', (latent_dim, dim_b, init1)),
                                            ('g', (latent_dim, dim_b, init1)), ('out', (dim_a, latent_dim, init2))):
                inputs.append(self._make_param('%s_%s_w' % (name, part), [dout, din, 1, 1, 1],
                                               init.get('weight_init') or ('XavierFill', {}), True))
                if not init.get('no_bias', 0):
                    inputs.append(self._make_param('%s_%s_b' % (name, part), [dout],
                                                   init.get('bias_init') or ('ConstantFill', {'value': 0.}), False))
            outputs += [name + '_theta', name + '_affinity_prob', name + '_y', name + '_out', name + '_sum']
        outs = self.net.FboNLStack(inputs, outputs, prefix=prefix, dim_a=int(dim_a), dim_b=int(dim_b),
                                   latent_dim=int(latent_dim), num_feat2=int(num_feat2), num_layers=int(num_layers),
                                   scale=float(scale), pre_act_ln=bool(pre_act_ln), ratio=float(dropout_ratio),
                                   no_bias=[int(bool(i.get('no_bias', 0))) for i in (init1, init1, init1, init2)])
        return outs[-1]

    # ---- parameter-free layers -------------------------------------------------
    def MaxPool(self, blob_in, blob_out, kernels=None, strides=None, pads=None, **kwargs):
        return self.net.MaxPool(blob_in, blob_out, kernels=list(kernels), strides=list(strides or [1] * len(kernels)),
                                pads=list(pads or [0] * 2 * len(kernels)))

    def AveragePool(self, blob_in, blob_out, kernels=None, strides=None, pads=None, **kwargs):
        return self.net.AveragePool(blob_in, blob_out, kernels=list(kernels),
                                    strides=list(strides or [1] * len(kernels)),
                                    pads=list(pads or [0] * 2 * len(kernels)))

    def Relu(self, blob_in, blob_out, **kwargs):
        return self.net.Relu(blob_in, blob_out)

    def Sigmoid(self, blob_in, blob_out, **kwargs):
        return self.net.Sigmoid(blob_in, blob_out)

    def Softmax(self, blob_in, blob_out, axis=1, **kwargs):
        return self.net.Softmax(blob_in, blob_out, axis=axis)

    def Scale(self, blob_in, blob_out, scale=1.0, **kwargs):
        return self.net.Scale(blob_in, blob_out, scale=float(scale))

    def Dropout(self, blob_in, blob_out, ratio=0.5, is_test=False, **kwargs):
        return self.net.Dropout(blob_in, blob_out, ratio=float(ratio), is_test=bool(is_test))

    def Transpose(self, blob_in, blob_out, axes=None, **kwargs):
        return self.net.Transpose(blob_in, blob_out, axes=tuple(axes))

    def Squeeze(self, blob_in, blob_out, dims=None, **kwargs):
        return self.net.Squeeze(blob_in, blob_out, dims=list(dims))

    def StopGradient(self, blob_in, blob_out, **kwargs):
        return self.net.StopGradient(blob_in, blob_out)

    def Reshape(self, blob_in, blob_out, shape=None, **kwargs):
        """Reshape(x, [y, old_shape], shape=...) or Reshape([x, shape_blob], [y, old_shape])
        (nonlocal_helper.py:80-83,125-128).  Returns (y, old_shape)."""
        args = {} if shape is None else {'shape': tuple(shape)}
        return self.net.Reshape(_as_list(blob_in), _as_list(blob_out), **args)

    def LayerNorm(self, blob_in, blob_out, axis=1, epsilon=1e-5, **kwargs):
        """LayerNorm(x, [y, mean, std]) (lfb_helper.py:163-166).  Returns the 3 outputs."""
        return self.net.LayerNorm(blob_in, _as_list(blob_out), axis=axis, epsilon=float(epsilon))

    def RoIAlign(self, blobs_in, blobs_out, pooled_w=7, pooled_h=7, spatial_scale=1.0, sampling_ratio=0, **kwargs):
        return self.net.RoIAlign(_as_list(blobs_in), _as_list(blobs_out), pooled_w=int(pooled_w),
                                 pooled_h=int(pooled_h), spatial_scale=float(spatial_scale),
                                 sampling_ratio=int(sampling_ratio))

    def SigmoidCrossEntropyLoss(self, blobs_in, blobs_out, scale=1.0, **kwargs):
        return self.net.SigmoidCrossEntropyLoss(_as_list(blobs_in), _as_list(blobs_out), scale=float(scale))

    def SoftmaxWithLoss(self, blobs_in, blobs_out, scale=1.0, **kwargs):
        return self.net.SoftmaxWithLoss(_as_list(blobs_in), _as_list(blobs_out), scale=float(scale))

    def WeightedSum(self, blobs_in, blob_out, **kwargs):
        return self.net.WeightedSum(_as_list(blobs_in), blob_out)

    def DequeueBlobs(self, queue_name, blob_names, **kwargs):
        return self.net.DequeueBlobs([queue_name], list(blob_names))

    def __getattr__(self, op_type):
        if op_type.startswith('_') or op_type in ('net', 'param_init_net'):
            raise AttributeError(op_type)
        return getattr(self.net, op_type)
