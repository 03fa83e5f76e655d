"""Inference-time graph surgery for the PyTorch/cuDNN stages around the hot path (they stay PyTorch calls):
eval-mode BatchNorm folded into the preceding convolution, ResNet trunks run channels-last so cuDNN's NHWC
tensor-core kernels need no per-layer NCHW<->NHWC conversion.  Applied AFTER weights are loaded
(`CUTIE.optimize_for_inference()`); the state_dict layout of an optimised model is no longer the checkpoint's."""
import contextlib

import torch
import torch.nn as nn
import torch.nn.functional as F  # noqa: F401


def fold_conv_bn(conv: nn.Conv2d, bn: nn.BatchNorm2d) -> nn.Conv2d:
    scale = bn.weight.detach() / torch.sqrt(bn.running_var.detach() + bn.eps)
    fused = nn.Conv2d(conv.in_channels, conv.out_channels, conv.kernel_size, conv.stride, conv.padding,
                      conv.dilation, conv.groups, bias=True).to(conv.weight.device, conv.weight.dtype)
    fused.weight.data = conv.weight.detach() * scale.view(-1, 1, 1, 1)
    bias = bn.bias.detach() - bn.running_mean.detach() * scale
    if conv.bias is not None:
        bias = bias + conv.bias.detach() * scale
    fused.bias.data = bias
    return fused


def fold_trunk_(module: nn.Module) -> int:
    """Folds every (convN, bnN) pair and (downsample.0, downsample.1) pair found under `module`, in place."""
    n = 0
    for m in module.modules():
        for i in (1, 2, 3):
            conv, bn = getattr(m, f'conv{i}', None), getattr(m, f'bn{i}', None)
            if isinstance(conv, nn.Conv2d) and isinstance(bn, nn.BatchNorm2d):
                setattr(m, f'conv{i}', fold_conv_bn(conv, bn))
                setattr(m, f'bn{i}', nn.Identity())
                n += 1
        ds = getattr(m, 'downsample', None)
        if isinstance(ds, nn.Sequential) and len(ds) == 2 and isinstance(ds[1], nn.BatchNorm2d):
            m.downsample = nn.Sequential(fold_conv_bn(ds[0], ds[1]), nn.Identity())
            n += 1
        if all(isinstance(getattr(m, f'bn{i}', nn.Identity()), nn.Identity) for i in (1, 2, 3)) and \
                isinstance(getattr(m, 'conv1', None), nn.Conv2d):
            m.bn_folded = True          # _Residual / encoder stems switch to the fused-epilogue forward
    return n


# ---------------------------------------------------------------------------------------------------
# convolution epilogues: bias (+ residual) (+ ReLU) without ATen's extra launches
# ---------------------------------------------------------------------------------------------------
class ConvEpilogueFuser:
    """`act(conv(x) + bias [+ z])` in fewer launches than PyTorch's convolution + broadcast bias add [+ add] [+ clamp].

    Unfused, a frame issues ~180 such epilogue launches: `elementwise_kernel<add>` for the bias adds (ATen runs them
    through a broadcast TensorIterator with no vector accesses), `clamp_scalar` for the ReLUs and the residual adds.  The convolutions themselves stay cuDNN calls (BASELINE.json north_star); three forms of the epilogue:

      'aten'    F.conv2d(x, w, b) [+ y.add_(z)] [+ relu_]                -- what PyTorch does; the reference form
      'cudnn'   torch.cudnn_convolution_add_relu(x, w, z, alpha, b, ..)  -- cuDNN's fused conv-bias-add-ReLU graph (the
                op PyTorch's own frozen-graph pass emits); ReLU epilogues only
      'kernel'  F.conv2d(x, w, None) + cutie_bias_act(y, b, z, relu)     -- the bias-less convolution followed by ONE
                float4 stream of ours (csrc/pixel.cu), same association as 'aten' => bit-identical results
      'pool'    (ResNet stems) bias-less convolution + cutie_bias_relu_maxpool: bias, clamp and 3x3/s2 pooling in one pass
      'tc'      cutie_conv_tc: the convolution ITSELF on the tensor cores (wgmma implicit GEMM, 3xTF32 operand split =
                fp32-class accuracy; csrc/conv_tc.cu) with bias, residual, ReLU and the ReLU of the INPUT in the same
                kernel -- 3x3 / stride 1 / pad 1 and 1x1 / stride 1 or 2 layers with Cin % 32 == 0 and Cout >= 64, dense
                NCHW or channels-last (the output keeps the input's memory format): SURVEY.md section 8(f).1-3 --
                PixelFFN, fuser, key projection, decoder, sensory update and the trunks' bottleneck convolutions
      'tc16'    cutie_conv_tc_f16: the same kernel with FP16 operands and fp32 accumulation -- what fp16 autocast asks of a
                convolution; taken instead of 'tc' only in AMP MODE (`amp_mode()`, entered by InferenceCore.step under
                autocast), except by layers marked `amp_fp32` (the sensory updaters' transforms, which the reference
                itself runs in autocast(enabled=False))

    DETERMINISTIC: the form is a function of the layer geometry, the epilogue and the mode alone -- `RULE`: eligible 3x3 / 1x1
    layers take 'tc' ('tc16' in amp mode); of the rest ReLU epilogues take 'cudnn', bias-only and bias+residual epilogues take 'kernel', stems take 'pool' -- (a committed choice, not re-timed per GPU); nothing is timed at run time, so two runs of the
    same video execute the same arithmetic.  CPU tensors (the oracle harness borrowing these modules) always take 'aten'.

    `cudnn_convolution_relu` hands the *uninitialised* output to cuDNN as the residual operand with alpha = 0;
    0 x (stale NaN bits) is NaN, so the no-residual case passes a persistent zero tensor of the output shape
    instead (read once per call, ~100 MB per 480p frame over all layers: 15 us of HBM time).
    """
    FORMS = ('aten', 'cudnn', 'kernel', 'tc', 'tc16')
    RULE = {'conv': 'tc', 'relu': 'cudnn', 'linear': 'kernel', 'stem': 'pool'}

    def __init__(self, enabled: bool = True, rule=None):
        self.enabled = enabled
        self.rule = dict(self.RULE if rule is None else rule)
        self.amp = False             # amp mode: eligible 'tc' layers take 'tc16' (amp_mode())
        self.counts = {}             # form -> number of distinct (layer, geometry, epilogue) triples routed to it
        self._seen = set()
        self._zeros = {}
        self._images = {}            # id(conv) -> (weight identity, operand image, counters) of the 'tc' form
        self._images16 = {}          # ... of the 'tc16' form

    @contextlib.contextmanager
    def amp_mode(self, on: bool = True):
        """Within the block eligible layers take the FP16-operand form 'tc16' (layers marked `amp_fp32` keep 'tc')."""
        prev, self.amp = self.amp, bool(on)
        try:
            yield self
        finally:
            self.amp = prev

    # -- the forms ------------------------------------------------------------------------------------
    @staticmethod
    def _conv(conv: nn.Conv2d, x: torch.Tensor, with_bias: bool) -> torch.Tensor:
        # nn.Conv2d's own convolution (class method: instances may carry a patched _conv_forward, and ObjConv2d
        # overrides forward for 5-D object tensors)
        return nn.Conv2d._conv_forward(conv, x, conv.weight, conv.bias if with_bias else None)

    @classmethod
    def unfused(cls, conv: nn.Conv2d, x: torch.Tensor, z=None, relu: bool = True, relu_in: bool = False) -> torch.Tensor:
        """The 'aten' form."""
        y = cls._conv(conv, F.relu(x) if relu_in else x, True)
        if z is not None:
            y = y.add_(z) if not y.requires_grad else y + z
        if relu:
            y = torch.relu_(y) if not y.requires_grad else torch.relu(y)
        return y

    def _zero_like_output(self, conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
        n, _, h, w = x.shape
        ho = (h + 2 * conv.padding[0] - conv.dilation[0] * (conv.kernel_size[0] - 1) - 1) // conv.stride[0] + 1
        wo = (w + 2 * conv.padding[1] - conv.dilation[1] * (conv.kernel_size[1] - 1) - 1) // conv.stride[1] + 1
        cl = x.is_contiguous(memory_format=torch.channels_last) and not x.is_contiguous()
        cl = cl or conv.weight.is_contiguous(memory_format=torch.channels_last) and not conv.weight.is_contiguous()
        key = (n, conv.out_channels, ho, wo, x.dtype, x.device, bool(cl))
        buf = self._zeros.get(key)
        if buf is None:
            buf = torch.empty(n, conv.out_channels, ho, wo, dtype=x.dtype, device=x.device,
                              memory_format=torch.channels_last if cl else torch.contiguous_format).zero_()
            self._zeros[key] = buf
        return buf

    def fused(self, conv: nn.Conv2d, x: torch.Tensor, z=None) -> torch.Tensor:
        """The 'cudnn' form (always with ReLU)."""
        if z is None:
            return torch.cudnn_convolution_add_relu(x, conv.weight, self._zero_like_output(conv, x), 0.0, conv.bias,
                                                    conv.stride, conv.padding, conv.dilation, conv.groups)
        return torch.cudnn_convolution_add_relu(x, conv.weight, z, 1.0, conv.bias,
                                                conv.stride, conv.padding, conv.dilation, conv.groups)

    def kernel(self, conv: nn.Conv2d, x: torch.Tensor, z=None, relu: bool = True) -> torch.Tensor:
        """The 'kernel' form: bias-less convolution + cutie_bias_act."""
        from cutie_b200 import kernels as K_
        return K_.bias_act_(self._conv(conv, x, False), conv.bias, z, relu)

    def tensor_core(self, conv: nn.Conv2d, x: torch.Tensor, z=None, relu: bool = True, relu_in: bool = False,
                    f16: bool = False) -> torch.Tensor:
        """The 'tc' form ('tc16' with f16=True).  The operand image is rebuilt whenever the weight tensor is replaced or
        written."""
        from cutie_b200 import kernels as K_
        w = conv.weight
        try:
            ident = (w.data_ptr(), w._version)
        except RuntimeError:                       # inference tensors carry no version counter
            ident = (w.data_ptr(), None)
        images = self._images16 if f16 else self._images
        hit = images.get(id(conv))
        if hit is None or hit[0] != ident:
            # the layer's operand image and its own shared-tile counters (zero between launches; one layer never runs
            # twice at the same time, different layers may -- encoder look-ahead -- so counters are never shared)
            img = K_.conv_weight_image_f16(w) if f16 else K_.conv_weight_image(w)
            hit = (ident, img, torch.zeros(8192, dtype=torch.int32, device=w.device))
            images[id(conv)] = hit
        return (K_.conv_tc_f16 if f16 else K_.conv_tc)(x, hit[1], conv.bias, conv.out_channels, ksize=conv.kernel_size[0],
                                                       stride=conv.stride[0], residual=z, relu_in=relu_in, relu_out=relu,
                                                       counters=hit[2])

    def _tc_eligible(self, conv: nn.Conv2d, x: torch.Tensor, z) -> bool:
        from cutie_b200 import kernels as K_
        return (self.rule.get('conv') == 'tc'
                and K_.conv_tc_eligible(conv.weight, conv.stride, conv.padding, conv.dilation, conv.groups))

    def run(self, form: str, conv: nn.Conv2d, x: torch.Tensor, z=None, relu: bool = True, relu_in: bool = False) -> torch.Tensor:
        if form == 'tc':
            return self.tensor_core(conv, x, z, relu, relu_in)
        if form == 'tc16':
            return self.tensor_core(conv, x, z, relu, relu_in, f16=True)
        if relu_in:
            x = F.relu(x)
        if form == 'cudnn':
            return self.fused(conv, x, z)
        if form == 'kernel':
            return self.kernel(conv, x, z, relu)
        return self.unfused(conv, x, z, relu)

    def _eligible(self, conv: nn.Conv2d, x: torch.Tensor) -> bool:
        return (self.enabled and x.is_cuda and conv.bias is not None and conv.padding_mode == 'zeros'
                and x.dim() == 4 and x.dtype == torch.float32 and not torch.is_grad_enabled())

    def _note(self, form: str, conv, x, z, relu):
        key = (id(conv), tuple(x.shape), z is not None, bool(relu), form)
        if key not in self._seen:
            self._seen.add(key)
            self.counts[form] = self.counts.get(form, 0) + 1

    def __call__(self, conv: nn.Conv2d, x: torch.Tensor, z=None, relu: bool = True, relu_in: bool = False) -> torch.Tensor:
        if not self._eligible(conv, x):
            return self.unfused(conv, x, z, relu, relu_in)
        if self._tc_eligible(conv, x, z):
            form = 'tc16' if self.amp and not getattr(conv, 'amp_fp32', False) else 'tc'
        else:
            form = self.rule['relu'] if relu else self.rule['linear']
        self._note(form, conv, x, z, relu)
        return self.run(form, conv, x, z, relu, relu_in)

    # -- ResNet stem: relu(conv(x) + bias) -> max_pool2d(3, 2, 1) ---------------------------------------------
    def stem(self, conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
        """max_pool2d(relu(conv(x)), 3, stride=2, padding=1): the bias-less convolution followed by
        cutie_bias_relu_maxpool ('pool': bias, clamp and pooling in one pass over the convolution output; they commute
        with max, so the result is bit-identical), or the conv+ReLU rule followed by ATen's pooling."""
        if not self._eligible(conv, x):
            return F.max_pool2d(self.unfused(conv, x), 3, stride=2, padding=1)
        if self.rule['stem'] == 'pool':
            from cutie_b200 import kernels as K_
            self._note('pool', conv, x, None, True)
            return K_.bias_relu_maxpool(self._conv(conv, x, False), conv.bias)
        return F.max_pool2d(self(conv, x, None, True), 3, stride=2, padding=1)

    def __deepcopy__(self, memo):          # a copied model gets its own fuser with the same settings
        new = ConvEpilogueFuser(self.enabled, self.rule)          # (operand images are rebuilt lazily by the copy)
        memo[id(self)] = new
        return new

    def report(self) -> dict:
        """`layers`: form -> distinct (layer, geometry, epilogue) triples routed to it so far, amp steps' 'tc16' included."""
        return {'enabled': self.enabled, 'rule': dict(self.rule), 'layers': dict(self.counts)}


def attach_epilogue_fuser(module: nn.Module, fuser: 'ConvEpilogueFuser') -> int:
    """Hands `fuser` to every nn.Conv2d under `module` (plain attributes, not parameters / buffers / sub-modules, so
    state_dict and .to() are unaffected).  Per model, not process-wide: an un-optimised model keeps PyTorch's launches.
    Besides `epilogue_fuser` (read by conv_relu / conv_add_relu) each convolution's `_conv_forward` is pointed at the
    fuser, so plain `conv(x)` calls -- no ReLU behind them -- get their bias from the fuser's choice as well."""
    n = 0
    for m in module.modules():
        if isinstance(m, nn.Conv2d):
            object.__setattr__(m, 'epilogue_fuser', fuser)
            object.__setattr__(m, '_conv_forward', _BiasOnlyForward(m, fuser))
            n += 1
    return n


class _BiasOnlyForward:
    """Instance-level replacement of nn.Conv2d._conv_forward(input, weight, bias) (called by Conv2d.forward)."""

    def __init__(self, conv: nn.Conv2d, fuser: ConvEpilogueFuser):
        self.conv, self.fuser = conv, fuser

    def __call__(self, x, weight, bias):
        conv = self.conv
        if bias is None or weight is not conv.weight or bias is not conv.bias:
            return nn.Conv2d._conv_forward(conv, x, weight, bias)
        return self.fuser(conv, x, None, relu=False)

    def __deepcopy__(self, memo):          # a copied module must point at ITS convolution (already in memo) and fuser
        import copy
        return _BiasOnlyForward(copy.deepcopy(self.conv, memo), copy.deepcopy(self.fuser, memo))


def conv_relu(conv: nn.Conv2d, x: torch.Tensor, relu_in: bool = False) -> torch.Tensor:
    """relu(conv(x)) (conv(relu(x)) inside if relu_in) -- in the form the model's fuser names for this layer, else
    convolution + bias add + clamp."""
    f = getattr(conv, 'epilogue_fuser', None)
    return ConvEpilogueFuser.unfused(conv, x, relu_in=relu_in) if f is None else f(conv, x, relu_in=relu_in)


def conv_relu_maxpool(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """max_pool2d(relu(conv(x)), 3, stride=2, padding=1) -- the ResNet stem."""
    f = getattr(conv, 'epilogue_fuser', None)
    if f is None:
        return F.max_pool2d(ConvEpilogueFuser.unfused(conv, x), 3, stride=2, padding=1)
    return f.stem(conv, x)


def conv_add(conv: nn.Conv2d, x: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """conv(x) + z (bias included, no activation): the closing convolution of a pre-activation residual block."""
    f = getattr(conv, 'epilogue_fuser', None)
    return ConvEpilogueFuser.unfused(conv, x, z, relu=False) if f is None else f(conv, x, z, relu=False)


def conv_plain(conv: nn.Conv2d, x: torch.Tensor) -> torch.Tensor:
    """conv(x) on a 4-D tensor for any nn.Conv2d subclass (ObjConv2d's own forward expects 5-D object tensors)."""
    f = getattr(conv, 'epilogue_fuser', None)
    return ConvEpilogueFuser._conv(conv, x, True) if f is None else f(conv, x, None, relu=False)


def conv_add_relu(conv: nn.Conv2d, x: torch.Tensor, z: torch.Tensor) -> torch.Tensor:
    """relu(conv(x) + z)."""
    f = getattr(conv, 'epilogue_fuser', None)
    return ConvEpilogueFuser.unfused(conv, x, z) if f is None else f(conv, x, z)
