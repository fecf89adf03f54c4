"""PyTorch autograd layers on the C ABI -- the role of tinycudann's `modules.py` (bindings/torch/tinycudann/modules.py:132-330).

    import tcnn_b200.torch_modules as tcnn
    model = tcnn.NetworkWithInputEncoding(n_input_dims=3, n_output_dims=3, encoding_config=enc, network_config=net)
    y = model(x)                      # x: [B, n_input_dims] float CUDA tensor -> [B, n_output_dims] fp16
    loss.backward(); torch_optimizer.step()   # model.params is a torch.nn.Parameter (fp32), as in tinycudann
    enc = tcnn.Encoding(3, enc_config)        # the grid encoding on its own (modules.py:312-330), fp16 features
    net = tcnn.Network(32, 3, net_config)     # the network on its own (modules.py:248-268)

Same conventions as the reference binding: parameters are an fp32 `torch.nn.Parameter` initialised by
`Module::initialize_params(seed)`, cast to fp16 for every call (modules.py:227-231); the batch is padded to the granularity of
256 (modules.py:222-226); gradients w.r.t. the output are multiplied by the loss scale (128 for fp16) before the native
backward pass and the parameter / input gradients divided by it afterwards (modules.py:166-171); the padded output columns are
sliced away (modules.py:233). Gradients w.r.t. the input positions are delivered when the input requires grad (modules.py:153-160).
Second-order terms (modules.py:161-200): the backward pass of `Encoding` is itself differentiable under `create_graph=True` for the
grid encodings (an eikonal loss on dL/dx reaches the grid table, the input and dL/d(output)); other encodings raise
"... does not support double backward". The network modules deliver first-order gradients only.

This file is glue: the work happens in libtcnn_b200 (fused sm_90a kernels) behind `tcnnb_module_*`, `tcnnb_encoding_*`, `tcnnb_network_*`.
"""
import torch

from . import Encoding as _NativeEncoding
from . import Module as _NativeModule
from . import Network as _NativeNetwork
from . import load

_BATCH_GRANULARITY = 256


class _ModuleFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, native, inputs, params, loss_scale):
        ctx.set_materialize_grads(False)
        output = native.fwd(inputs, params)
        ctx.save_for_backward(inputs, params, output)
        ctx.native = native
        ctx.loss_scale = loss_scale
        return output

    @staticmethod
    def backward(ctx, doutput):
        if doutput is None:
            return None, None, None, None
        inputs, params, output = ctx.saved_tensors
        want_input, want_params = ctx.needs_input_grad[1], ctx.needs_input_grad[2]
        if not (want_input or want_params):
            return None, None, None, None
        if isinstance(ctx.native, _NativeEncoding) and torch.is_grad_enabled():
            # backward with create_graph=True: the gradients become differentiable (a loss on dL_dinput, e.g. an eikonal term)
            dinput, grads = _EncodingBackwardFunction.apply(ctx.native, ctx.loss_scale, doutput, inputs, params, want_input, want_params)
            return None, dinput, grads, None
        with torch.no_grad():
            scaled = (doutput.to(torch.float32) * ctx.loss_scale).to(torch.float16).contiguous()
            if isinstance(ctx.native, _NativeEncoding):
                grads, dinput = ctx.native.bwd(inputs, params, scaled, want_params=want_params, want_input=want_input)
            elif want_input:
                grads, dinput = ctx.native.bwd(inputs, params, scaled, output=output, want_input_grad=True, want_param_grad=want_params)
            else:
                grads, dinput = ctx.native.bwd(inputs, params, scaled, output=output), None
            grads = (grads.to(torch.float32) / ctx.loss_scale).to(params.dtype) if grads is not None else None
            dinput = (dinput / ctx.loss_scale).to(inputs.dtype) if dinput is not None else None
        return None, dinput, grads, None


class _EncodingBackwardFunction(torch.autograd.Function):
    """The encoding's backward pass as a differentiable function of (doutput, inputs, params) -- modules.py:161-200. Its own backward
    is Module::backward_backward_input: grid encodings only, every other encoding raises "... does not support double backward"."""

    @staticmethod
    def forward(ctx, native, loss_scale, doutput, inputs, params, want_input, want_params):
        ctx.set_materialize_grads(False)
        scaled = (doutput.to(torch.float32) * loss_scale).to(torch.float16).contiguous()
        grads, dinput = native.bwd(inputs, params, scaled, want_params=want_params, want_input=want_input)
        grads = (grads.to(torch.float32) / loss_scale).to(params.dtype) if grads is not None else None
        dinput = (dinput / loss_scale).to(inputs.dtype) if dinput is not None else None
        ctx.save_for_backward(inputs, params, scaled)
        ctx.native = native
        ctx.loss_scale = loss_scale
        return dinput, grads

    @staticmethod
    def backward(ctx, d_dinput, d_dparams):
        # d_dparams (a loss on the parameter gradient) is not propagated, as in the reference ("x d(dL_dparam)_d(...)")
        want_doutput, want_input, want_params = ctx.needs_input_grad[2], ctx.needs_input_grad[3], ctx.needs_input_grad[4]
        if d_dinput is None or not (want_doutput or want_input or want_params):
            return None, None, None, None, None, None, None
        inputs, params, scaled = ctx.saved_tensors
        with torch.no_grad():
            # dL_doutput reached the native call multiplied by the loss scale: the parameter and input results carry it, the
            # dL_doutput result (a function of d_dinput alone) does not
            ddoutput, grads, dinput = ctx.native.bwd_bwd_input(inputs, params, d_dinput.to(torch.float32).contiguous(), scaled,
                                                               want_doutput=want_doutput, want_params=want_params, want_input=want_input)
            grads = (grads.to(torch.float32) / ctx.loss_scale).to(params.dtype) if grads is not None else None
            dinput = (dinput / ctx.loss_scale).to(inputs.dtype) if dinput is not None else None
        return None, None, ddoutput, dinput, grads, None, None


class _TcnnModule(torch.nn.Module):
    def __init__(self, native, n_input_dims, n_output_dims, seed):
        super().__init__()
        self.native_tcnn_module = native
        self.n_input_dims = n_input_dims
        self.n_output_dims = n_output_dims
        self.seed = seed
        self.dtype = torch.float16
        self.params = torch.nn.Parameter(native.initial_params(seed), requires_grad=True)
        self.loss_scale = float(load().tcnnb_default_loss_scale())

    def forward(self, x):
        x = x.cuda() if not x.is_cuda else x
        batch = x.shape[0]
        padded = (batch + _BATCH_GRANULARITY - 1) // _BATCH_GRANULARITY * _BATCH_GRANULARITY
        x = x.to(torch.float32)
        if padded != batch:
            x = torch.nn.functional.pad(x, [0, 0, 0, padded - batch])
        out = _ModuleFunction.apply(self.native_tcnn_module, x.contiguous(), self.params.to(torch.float16).contiguous(), self.loss_scale)
        return out[:batch, : self.n_output_dims]

    def extra_repr(self):
        return f"n_input_dims={self.n_input_dims}, n_output_dims={self.n_output_dims}, seed={self.seed}, dtype={self.dtype}"


class NetworkWithInputEncoding(_TcnnModule):
    """tinycudann.NetworkWithInputEncoding (modules.py:270-310) for the HashGrid + FullyFusedMLP path."""

    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config, seed=1337):
        self.encoding_config = encoding_config
        self.network_config = network_config
        super().__init__(_NativeModule(n_input_dims, n_output_dims, encoding_config, network_config), n_input_dims, n_output_dims, seed)


class Encoding(_TcnnModule):
    """tinycudann.Encoding (modules.py:312-330): grids, Identity, Frequency, TriangleWave, OneBlob, SphericalHarmonics, Empty, Composite
    (Concatenation / Sum / Product, dims_to_encode_begin) and the NRC shorthand; fp16 features."""

    def __init__(self, n_input_dims, encoding_config, seed=1337):
        self.encoding_config = encoding_config
        native = _NativeEncoding(n_input_dims, encoding_config)
        super().__init__(native, n_input_dims, native.n_output_dims, seed)


class _NetworkAdapter:
    """The stand-alone network behind the same fwd / bwd / initial_params surface as the other native modules (fp32 inputs through the
    Identity encoding, cpp::create_network, src/cpp_api.cu:160-162)."""

    def __init__(self, native):
        self.native = native

    def initial_params(self, seed):
        return self.native.initial_params(seed)

    def fwd(self, inputs, params):
        return self.native.module_inference(inputs, params)

    def bwd(self, inputs, params, dL_doutput, output=None, want_input_grad=False, want_param_grad=True):
        dinput, grads = self.native.module_backward(inputs, dL_doutput, params, want_input_grad=want_input_grad, want_param_grad=want_param_grad)
        return (grads, dinput) if want_input_grad else grads


class Network(_TcnnModule):
    """tinycudann.Network (modules.py:248-268): fp32 inputs through the Identity encoding -> fp16 outputs, with autograd w.r.t. the
    parameters and the inputs (dgrad chain + weight-gradient kernels of the stand-alone network)."""

    def __init__(self, n_input_dims, n_output_dims, network_config, seed=1337):
        self.network_config = network_config
        native = _NativeNetwork(n_input_dims, n_output_dims, network_config)
        super().__init__(_NetworkAdapter(native), n_input_dims, n_output_dims, seed)
