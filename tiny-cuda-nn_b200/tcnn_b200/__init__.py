"""tcnn_b200 -- thin ctypes binding over the C ABI in include/tcnn_b200.h (libtcnn_b200.so).

This mirrors, in Python, the names a user of the reference touches on this path:
`create_from_config(n_input_dims, n_output_dims, config)` -> TrainableModel with `.trainer.training_step(...)`,
`.trainer.loss()`, `.network.inference(...)` (config.h:46-63, trainer.h:254-378, object.h:214).
It is plumbing for tests and bench.py: torch is used only for device memory and streams. There is no CPU
fallback -- if the CUDA library is missing or the device is not an sm_90 (H100-class) GPU, construction raises.
"""
import ctypes
import json
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
# TCNNB_LIB selects another build of the same library (profiling experiments use an ABLATION=1 build next to the product one)
_LIB_PATH = os.environ.get("TCNNB_LIB") or os.path.join(os.path.dirname(_HERE), "libtcnn_b200.so")
_lib = None


class TcnnError(RuntimeError):
    pass


class DebugTaps(ctypes.Structure):
    _fields_ = [
        ("encoded", ctypes.c_void_p),
        ("hidden", ctypes.c_void_p),
        ("output", ctypes.c_void_p),
        ("dL_doutput", ctypes.c_void_p),
        ("grad_hidden", ctypes.c_void_p),
        ("dL_dencoded", ctypes.c_void_p),
        ("loss_values", ctypes.c_void_p),
    ]


# (name, restype, argtypes) of every symbol include/tcnn_b200.h declares; tests check the .so exports all of them.
_u32, _u64, _f32p, _vp, _int = ctypes.c_uint32, ctypes.c_uint64, ctypes.POINTER(ctypes.c_float), ctypes.c_void_p, ctypes.c_int
ABI = [
    ("tcnnb_last_error", ctypes.c_char_p, []),
    ("tcnnb_batch_size_granularity", _u32, []),
    ("tcnnb_default_loss_scale", ctypes.c_float, []),
    ("tcnnb_cuda_device", _int, []),
    ("tcnnb_set_cuda_device", _int, [_int]),
    ("tcnnb_abi_version", _u32, []),
    ("tcnnb_create_from_config", _int, [_u32, _u32, ctypes.c_char_p, _u32, ctypes.POINTER(_vp)]),
    ("tcnnb_destroy", None, [_vp]),
    ("tcnnb_n_params_padded", ctypes.c_uint64, [_vp]),
    ("tcnnb_n_params", _u64, [_vp]),
    ("tcnnb_n_mlp_params", _u64, [_vp]),
    ("tcnnb_n_input_dims", _u32, [_vp]),
    ("tcnnb_n_output_dims", _u32, [_vp]),
    ("tcnnb_padded_output_width", _u32, [_vp]),
    ("tcnnb_encoded_width", _u32, [_vp]),
    ("tcnnb_params_full_precision", _vp, [_vp]),
    ("tcnnb_params", _vp, [_vp]),
    ("tcnnb_params_inference", _vp, [_vp]),
    ("tcnnb_param_gradients", _vp, [_vp]),
    ("tcnnb_grid_levels", _int, [_vp, ctypes.POINTER(_u32), ctypes.POINTER(_u32), _f32p, ctypes.POINTER(_u32)]),
    ("tcnnb_hyperparams", ctypes.c_char_p, [_vp]),
    ("tcnnb_set_params_full_precision", _int, [_vp, _vp, _u64, _int]),
    ("tcnnb_set_params", _int, [_vp, _vp, _u64, _int]),
    ("tcnnb_optimizer_state", _int, [_vp, ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_vp), ctypes.POINTER(_u32), _f32p]),
    ("tcnnb_set_optimizer_progress", _int, [_vp, _u32, ctypes.c_float]),
    ("tcnnb_training_step", _int, [_vp, _vp, _u32, _vp, _vp, _int]),
    ("tcnnb_training_step_shard", _int, [_vp, _vp, _u32, _u32, _vp, _vp, _int]),
    ("tcnnb_optimizer_step", _int, [_vp, _vp]),
    ("tcnnb_generate_random_uniform", _int, [_vp, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint64, _vp, ctypes.c_float, ctypes.c_float]),
    ("tcnnb_module_create", _int, [ctypes.c_uint32, ctypes.c_uint32, ctypes.c_char_p, ctypes.c_char_p, ctypes.POINTER(_vp)]),
    ("tcnnb_module_initialize_params", _int, [_vp, ctypes.c_uint64, _vp, ctypes.c_float]),
    ("tcnnb_module_inference", _int, [_vp, _vp, ctypes.c_uint32, _vp, _vp, _vp]),
    ("tcnnb_module_forward", _int, [_vp, _vp, ctypes.c_uint32, _vp, _vp, _vp, ctypes.c_int]),
    ("tcnnb_module_backward", _int, [_vp, _vp, ctypes.c_uint32, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("tcnnb_encoding_create", _int, [_u32, ctypes.c_char_p, ctypes.POINTER(_vp)]),
    ("tcnnb_encoding_destroy", None, [_vp]),
    ("tcnnb_encoding_n_params", _u64, [_vp]),
    ("tcnnb_encoding_n_input_dims", _u32, [_vp]),
    ("tcnnb_encoding_n_output_dims", _u32, [_vp]),
    ("tcnnb_encoding_grid_levels", _int, [_vp, ctypes.POINTER(_u32), ctypes.POINTER(_u32), _f32p, ctypes.POINTER(_u32)]),
    ("tcnnb_encoding_set_max_level", _int, [_vp, ctypes.c_float]),
    ("tcnnb_encoding_initialize_params", _int, [_vp, _u64, _vp, ctypes.c_float]),
    ("tcnnb_encoding_forward", _int, [_vp, _vp, _u32, _vp, _vp, _vp]),
    ("tcnnb_encoding_backward", _int, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    ("tcnnb_network_create", _int, [_u32, _u32, ctypes.c_char_p, ctypes.POINTER(_vp)]),
    ("tcnnb_network_destroy", None, [_vp]),
    ("tcnnb_network_n_params", _u64, [_vp]),
    ("tcnnb_network_input_width", _u32, [_vp]),
    ("tcnnb_network_padded_output_width", _u32, [_vp]),
    ("tcnnb_network_width", _u32, [_vp]),
    ("tcnnb_network_n_hidden_layers", _u32, [_vp]),
    ("tcnnb_network_initialize_params", _int, [_vp, _u64, _vp, ctypes.c_float]),
    ("tcnnb_network_inference_mixed_precision", _int, [_vp, _vp, _u32, _vp, _vp, _vp]),
    ("tcnnb_network_forward", _int, [_vp, _vp, _u32, _vp, _vp, _vp, _vp]),
    ("tcnnb_network_backward", _int, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp, _vp, _vp]),
    ("tcnnb_network_module_backward", _int, [_vp, _vp, _u32, _vp, _vp, _vp, _vp, _vp]),
    ("tcnnb_network_inference", _int, [_vp, _vp, _u32, _vp, _vp, _vp]),
    ("tcnnb_network_debug_clocks", _int, [_vp, _vp]),
    ("tcnnb_network_module_inference", _int, [_vp, _vp, _u32, _vp, _vp, _vp]),
    ("tcnnb_dp_unique_id", _int, [_vp, ctypes.c_uint64]),
    ("tcnnb_dp_init", _int, [_vp, _vp, _vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]),
    ("tcnnb_dp_shards_optimizer", _int, [_vp]),
    ("tcnnb_dp_attach_symmetric", _int, [_vp, ctypes.POINTER(ctypes.c_uint64), ctypes.c_uint64, ctypes.c_uint64]),
    ("tcnnb_dp_engine", _int, [_vp]),
    ("tcnnb_dp_training_step", _int, [_vp, _vp, ctypes.c_uint32, ctypes.c_uint32, _vp, _vp]),
    ("tcnnb_dp_sync_full_precision", _int, [_vp, _vp]),
    ("tcnnb_dp_finish", _int, [_vp]),
    ("tcnnb_wait_before_compute", _int, [_vp, _vp]),
    ("tcnnb_optimizer_step_ranges", _int, [_vp, _vp, ctypes.c_uint32, ctypes.POINTER(ctypes.c_uint64), ctypes.POINTER(ctypes.c_uint64)]),
    ("tcnnb_mlp_gradient_accumulator", _vp, [_vp]),
    ("tcnnb_grid_gradients", _vp, [_vp]),
    ("tcnnb_loss", _int, [_vp, _vp, _f32p]),
    ("tcnnb_inference", _int, [_vp, _vp, _u32, _vp, _vp]),
    ("tcnnb_training_step_host", _int, [_vp, _u32, _vp, _vp, _f32p]),
    ("tcnnb_training_step_host_submit", _int, [_vp, _u32, _vp, _vp, ctypes.POINTER(_u64)]),
    ("tcnnb_training_step_host_wait", _int, [_vp, _u64, _f32p]),
    ("tcnnb_dp_training_step_host_submit", _int, [_vp, _u32, _u32, _vp, _vp, ctypes.POINTER(_u64)]),
    ("tcnnb_inference_host", _int, [_vp, _u32, _vp, _vp]),
    ("tcnnb_serialize_size", _u64, [_vp, _int]),
    ("tcnnb_serialize", _int, [_vp, _vp, _u64, _int]),
    ("tcnnb_deserialize", _int, [_vp, _vp, _u64]),
    ("tcnnb_set_debug_taps", _int, [_vp, ctypes.POINTER(DebugTaps)]),
    ("tcnnb_debug_set", _int, [_vp, ctypes.c_char_p, _int]),
    ("tcnnb_set_profiling", _int, [_vp, _int]),
    ("tcnnb_read_profile", _int, [_vp, _f32p, _f32p, _f32p, ctypes.POINTER(_u32)]),
    ("tcnnb_kernel_launch_count", _u64, []),
]


def lib_path():
    return _LIB_PATH


def load():
    """Load libtcnn_b200.so (fails loudly if it has not been built: `python __graft_entry__.py build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(_LIB_PATH):
        raise TcnnError(f"{_LIB_PATH} is missing: build the CUDA extension first (python __graft_entry__.py build). There is no CPU fallback.")
    import torch  # noqa: F401  -- makes libcudart.so.12 resident before our library resolves it

    lib = ctypes.CDLL(_LIB_PATH)
    for name, restype, argtypes in ABI:
        fn = getattr(lib, name)
        fn.restype = restype
        fn.argtypes = argtypes
    _lib = lib
    return lib


def _check(rc):
    if rc != 0:
        raise TcnnError(load().tcnnb_last_error().decode())


def _stream_handle(stream):
    if stream is None:
        import torch

        return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)
    if isinstance(stream, int):
        return ctypes.c_void_p(stream)
    return ctypes.c_void_p(stream.cuda_stream)


class _Network:
    """NetworkWithInputEncoding surface: inference / n_params / padded_output_width."""

    def __init__(self, model):
        self._m = model

    def n_params(self):
        return self._m.n_params

    def padded_output_width(self):
        return load().tcnnb_padded_output_width(self._m._h)

    def inference(self, inputs, outputs=None, stream=None):
        """network->inference(stream, input, output): inputs [B, n_in] fp32 cuda -> [B, n_out] fp32 (object.h:214)."""
        import torch

        m = self._m
        assert inputs.is_cuda and inputs.dtype == torch.float32 and inputs.is_contiguous()
        B = inputs.shape[0]
        if outputs is None:
            outputs = torch.empty(B, m.n_output_dims, dtype=torch.float32, device=inputs.device)
        _check(load().tcnnb_inference(m._h, _stream_handle(stream), B, inputs.data_ptr(), outputs.data_ptr()))
        return outputs


class _Trainer:
    """Trainer surface: training_step / loss / params / param_gradients / serialize (trainer.h)."""

    def __init__(self, model):
        self._m = model

    def training_step(self, inputs, targets, run_optimizer=True, stream=None):
        import torch

        m = self._m
        assert inputs.is_cuda and targets.is_cuda and inputs.dtype == torch.float32 and targets.dtype == torch.float32
        assert inputs.is_contiguous() and targets.is_contiguous()
        _check(load().tcnnb_training_step(m._h, _stream_handle(stream), inputs.shape[0], inputs.data_ptr(), targets.data_ptr(), int(run_optimizer)))
        return self

    def training_step_shard(self, inputs, targets, global_batch_size, run_optimizer=False, stream=None):
        m = self._m
        _check(load().tcnnb_training_step_shard(m._h, _stream_handle(stream), inputs.shape[0], global_batch_size, inputs.data_ptr(), targets.data_ptr(), int(run_optimizer)))
        return self

    def optimizer_step(self, stream=None, ranges=None):
        """Adam on the current gradients; `ranges` = [(begin, count), ...] restricts it to those parameter spans."""
        if ranges is None:
            _check(load().tcnnb_optimizer_step(self._m._h, _stream_handle(stream)))
            return
        n = len(ranges)
        b = (ctypes.c_uint64 * n)(*[int(r[0]) for r in ranges])
        c = (ctypes.c_uint64 * n)(*[int(r[1]) for r in ranges])
        _check(load().tcnnb_optimizer_step_ranges(self._m._h, _stream_handle(stream), n, b, c))

    def loss(self, ctx=None, stream=None):
        out = ctypes.c_float(0)
        _check(load().tcnnb_loss(self._m._h, _stream_handle(stream), ctypes.byref(out)))
        return out.value

    def n_params(self):
        return self._m.n_params

    def _view(self, ptr, n, dtype):
        import torch

        class _Ext:
            pass

        itemsize = torch.empty((), dtype=dtype).element_size()
        typestr = {torch.float32: "<f4", torch.float16: "<f2", torch.int32: "<i4"}[dtype]
        holder = _Ext()
        holder.__cuda_array_interface__ = {"shape": (n,), "typestr": typestr, "data": (ptr, False), "version": 2, "strides": (itemsize,)}
        return torch.as_tensor(holder, device="cuda")

    def params_full_precision(self):
        import torch

        return self._view(load().tcnnb_params_full_precision(self._m._h), self._m.n_params, torch.float32)

    def params(self):
        import torch

        return self._view(load().tcnnb_params(self._m._h), self._m.n_params, torch.float16)

    def params_inference(self):
        """Trainer::params_inference(): the Ema wrapper's averaged weights when the optimizer has one, else params()."""
        import torch

        return self._view(load().tcnnb_params_inference(self._m._h), self._m.n_params, torch.float16)

    def param_gradients(self):
        import torch

        ptr = load().tcnnb_param_gradients(self._m._h)
        if not ptr:
            raise TcnnError(load().tcnnb_last_error().decode())
        return self._view(ptr, self._m.n_params, torch.float16)

    def mlp_gradient_accumulator(self):
        import torch

        return self._view(load().tcnnb_mlp_gradient_accumulator(self._m._h), self._m.n_mlp_params, torch.float32)

    def gradient_buffers(self):
        """The two buffers a data-parallel all-reduce must sum: fp16 grid-gradient table, fp32 MLP weight-gradient accumulator."""
        if not hasattr(self, "_grad_bufs"):
            import torch

            # NOT tcnnb_param_gradients(): that call materialises the fp16 MLP gradients and re-arms the fp32 accumulator
            ptr = load().tcnnb_grid_gradients(self._m._h)
            self._grad_bufs = [self._view(ptr, self._m.n_params - self._m.n_mlp_params, torch.float16), self.mlp_gradient_accumulator()]
        return self._grad_bufs

    def sharded_buffers(self):
        """Whole (padded) parameter vector views for the sharded-optimizer trainer: fp16 gradients, fp16 working parameters,
        fp32 masters -- each n_params_padded long -- plus the real parameter count and the number of network weights."""
        if not hasattr(self, "_sharded"):
            import torch

            lib, h = load(), self._m._h
            n_pad = int(lib.tcnnb_n_params_padded(h))
            self._sharded = {
                "grads": self._view(lib.tcnnb_param_gradients(h), n_pad, torch.float16),
                "params": self._view(lib.tcnnb_params(h), n_pad, torch.float16),
                "masters": self._view(lib.tcnnb_params_full_precision(h), n_pad, torch.float32),
                "n_params": self._m.n_params,
                "n_matrix": self._m.n_mlp_params,
            }
        return self._sharded

    # ---- native data parallelism (NCCL inside libtcnn_b200; tcnn_b200/dp.py drives it)
    def dp_native_init(self, group, shard_optimizer=True):
        """Create this model's NCCL communicators across `group` (a torch.distributed NCCL group): two ids from rank 0."""
        import torch
        import torch.distributed as dist

        lib, h = load(), self._m._h
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        ids = torch.zeros(256, dtype=torch.uint8)
        if rank == 0:
            buf = (ctypes.c_char * 128)()
            for k in range(2):
                _check(lib.tcnnb_dp_unique_id(buf, 128))
                ids[128 * k : 128 * (k + 1)] = torch.frombuffer(bytearray(buf.raw), dtype=torch.uint8)
        ids = ids.cuda()
        dist.broadcast(ids, src=dist.get_global_rank(group, 0) if group is not None else 0, group=group)
        raw = bytes(ids.cpu().numpy().tobytes())
        _check(lib.tcnnb_dp_init(h, ctypes.c_char_p(raw[:128]), ctypes.c_char_p(raw[128:]), world, rank, int(bool(shard_optimizer))))
        return bool(lib.tcnnb_dp_shards_optimizer(h))

    def dp_symmetric_bytes(self):
        """Size of the symmetric buffer of the peer-memory engine: fp16 params + fp16 gradients (padded) + flags."""
        return 4 * int(load().tcnnb_n_params_padded(self._m._h)) + 256

    def dp_attach_symmetric(self, peer_ptrs, multicast_ptr, n_bytes):
        arr = (ctypes.c_uint64 * len(peer_ptrs))(*peer_ptrs)
        _check(load().tcnnb_dp_attach_symmetric(self._m._h, arr, ctypes.c_uint64(multicast_ptr), ctypes.c_uint64(n_bytes)))
        for cached in ("_sharded", "_grad_bufs"):  # views of the old parameter / gradient regions
            if hasattr(self, cached):
                delattr(self, cached)

    def dp_engine(self):
        return {0: "single", 1: "nccl", 2: "peer-memory-p2p", 3: "peer-memory-multicast"}[load().tcnnb_dp_engine(self._m._h)]

    def dp_training_step(self, inputs, targets, global_batch_size, stream=None):
        _check(load().tcnnb_dp_training_step(self._m._h, _stream_handle(stream), inputs.shape[0], global_batch_size, inputs.data_ptr(), targets.data_ptr()))

    def dp_sync_full_precision(self, stream=None):
        _check(load().tcnnb_dp_sync_full_precision(self._m._h, _stream_handle(stream)))

    def dp_finish(self):
        _check(load().tcnnb_dp_finish(self._m._h))

    def wait_before_compute(self, event):
        """The next kernel of this model that reads the parameters waits for `event` (a torch.cuda.Event, kept alive here)."""
        self._pending_event = event
        _check(load().tcnnb_wait_before_compute(self._m._h, ctypes.c_void_p(event.cuda_event)))

    def finalize_gradients(self):
        """Round the fp32 network weight-gradient sums into the fp16 gradient buffer (what the reference's buffer holds)."""
        if not load().tcnnb_param_gradients(self._m._h):
            raise TcnnError(load().tcnnb_last_error().decode())

    def device(self):
        return "cuda"

    def set_params_full_precision(self, params):
        import torch

        if params.is_cuda:
            _check(load().tcnnb_set_params_full_precision(self._m._h, params.data_ptr(), params.numel(), 1))
        else:
            p = params.contiguous().to(torch.float32)
            _check(load().tcnnb_set_params_full_precision(self._m._h, p.data_ptr(), p.numel(), 0))

    def set_params(self, params16):
        """trainer->set_params (trainer.h:423-440): fp16 working parameters; the fp32 masters follow."""
        import torch

        p = params16.contiguous().to(torch.float16)
        _check(load().tcnnb_set_params(self._m._h, p.data_ptr(), p.numel(), 1 if p.is_cuda else 0))

    def serialize(self, with_optimizer=False):
        n = load().tcnnb_serialize_size(self._m._h, int(with_optimizer))
        buf = (ctypes.c_char * n)()
        _check(load().tcnnb_serialize(self._m._h, buf, n, int(with_optimizer)))
        return bytes(buf)

    def deserialize(self, blob):
        buf = ctypes.create_string_buffer(blob, len(blob))
        _check(load().tcnnb_deserialize(self._m._h, buf, len(blob)))


class Pcg32:
    """Host-side state of tiny-cuda-nn's default_rng_t (PCG-XSH-RR 64/32, stream constant 1): what generate_random_uniform
    needs to know -- (state, inc) -- and the O(log n) jump-ahead that advances it past the numbers a fill has consumed."""

    MULT = 0x5851F42D4C957F2D
    MASK = (1 << 64) - 1

    def __init__(self, seed=1337, seq=1):
        self.state = 0
        self.inc = ((seq << 1) | 1) & self.MASK
        self._step()
        self.state = (self.state + seed) & self.MASK
        self._step()

    def _step(self):
        self.state = (self.state * self.MULT + self.inc) & self.MASK

    def advance(self, delta):
        cur_mult, cur_plus, acc_mult, acc_plus = self.MULT, self.inc, 1, 0
        while delta > 0:
            if delta & 1:
                acc_mult = (acc_mult * cur_mult) & self.MASK
                acc_plus = (acc_plus * cur_mult + cur_plus) & self.MASK
            cur_plus = ((cur_mult + 1) * cur_plus) & self.MASK
            cur_mult = (cur_mult * cur_mult) & self.MASK
            delta >>= 1
        self.state = (acc_mult * self.state + acc_plus) & self.MASK


def generate_random_uniform(rng, n, lower=0.0, upper=1.0, stream=None):
    """generate_random_uniform<float>(stream, rng, n, ptr, lower, upper) (random.h:56-69): n uniform numbers on the current CUDA
    device, the reference's sequence for this generator state; advances `rng` by n."""
    import torch

    out = torch.empty(n, dtype=torch.float32, device="cuda")
    _check(load().tcnnb_generate_random_uniform(_stream_handle(stream), ctypes.c_uint64(rng.state), ctypes.c_uint64(rng.inc), ctypes.c_uint64(n), ctypes.c_void_p(out.data_ptr()),
                                                ctypes.c_float(lower), ctypes.c_float(upper)))
    rng.advance(n)
    return out


class Module:
    """tcnn::cpp::Module for a network with input encoding (cpp_api.h:76-125): caller-owned parameters, fp16 in/out.

    Mirrors what bindings/torch/tinycudann/bindings.cpp hands to autograd: `fwd(input, params)` -> padded fp16 output,
    `bwd(input, params, dL_doutput)` -> fp16 dL_dparams, `initial_params(seed)` -> fp32 parameter vector."""

    def __init__(self, n_input_dims, n_output_dims, encoding_config, network_config):
        lib = load()
        handle = ctypes.c_void_p()
        enc = encoding_config if isinstance(encoding_config, str) else json.dumps(encoding_config)
        net = network_config if isinstance(network_config, str) else json.dumps(network_config)
        _check(lib.tcnnb_module_create(n_input_dims, n_output_dims, enc.encode(), net.encode(), ctypes.byref(handle)))
        self._h = handle
        self.n_input_dims = n_input_dims
        self.n_output_dims = lib.tcnnb_padded_output_width(handle)  # Module::n_output_dims() is the PADDED width (cpp_api.cu:137)
        self.n_params = lib.tcnnb_n_params(handle)

    def initial_params(self, seed=1337, scale=1.0):
        import torch

        p = torch.empty(self.n_params, dtype=torch.float32, device="cuda")
        _check(load().tcnnb_module_initialize_params(self._h, seed, ctypes.c_void_p(p.data_ptr()), ctypes.c_float(scale)))
        return p

    def fwd(self, inputs, params, stream=None, inference=False):
        import torch

        out = torch.empty(inputs.shape[0], self.n_output_dims, dtype=torch.float16, device="cuda")
        lib = load()
        if inference:
            _check(lib.tcnnb_module_inference(self._h, _stream_handle(stream), inputs.shape[0], inputs.data_ptr(), out.data_ptr(), params.data_ptr()))
        else:
            _check(lib.tcnnb_module_forward(self._h, _stream_handle(stream), inputs.shape[0], inputs.data_ptr(), out.data_ptr(), params.data_ptr(), 0))
        return out

    def bwd(self, inputs, params, dL_doutput, output=None, stream=None, want_input_grad=False, want_param_grad=True):
        """dL_dparams (fp16 [n_params]); with want_input_grad -> (dL_dparams or None, dL_dinput fp32 [n][n_input_dims])."""
        import torch

        grads = torch.empty(self.n_params, dtype=torch.float16, device="cuda") if want_param_grad else None
        dinput = torch.empty(inputs.shape[0], self.n_input_dims, dtype=torch.float32, device="cuda") if want_input_grad else None
        _check(load().tcnnb_module_backward(self._h, _stream_handle(stream), inputs.shape[0], dinput.data_ptr() if want_input_grad else None, dL_doutput.data_ptr(),
                                            grads.data_ptr() if want_param_grad else None, inputs.data_ptr(), output.data_ptr() if output is not None else None, params.data_ptr()))
        return (grads, dinput) if want_input_grad else grads

    def close(self):
        if self._h:
            load().tcnnb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class Encoding:
    """tcnn::cpp::create_encoding (cpp_api.h:124) for the grid encodings: caller-owned fp16 parameters, fp16 features."""

    def __init__(self, n_input_dims, encoding_config):
        lib = load()
        h = ctypes.c_void_p()
        text = encoding_config if isinstance(encoding_config, str) else json.dumps(encoding_config)
        _check(lib.tcnnb_encoding_create(n_input_dims, text.encode(), ctypes.byref(h)))
        self._h = h
        self.n_input_dims = n_input_dims
        self.n_params = lib.tcnnb_encoding_n_params(h)
        self.n_output_dims = lib.tcnnb_encoding_n_output_dims(h)

    def grid_levels(self):
        n = ctypes.c_uint32(0)
        offsets = (ctypes.c_uint32 * 129)()
        scales = (ctypes.c_float * 128)()
        res = (ctypes.c_uint32 * 128)()
        _check(load().tcnnb_encoding_grid_levels(self._h, ctypes.byref(n), offsets, scales, res))
        L = n.value
        return {"n_levels": L, "offsets": list(offsets[: L + 1]), "scales": list(scales[:L]), "resolutions": list(res[:L])}

    def set_max_level(self, value):
        _check(load().tcnnb_encoding_set_max_level(self._h, float(value)))

    def initial_params(self, seed=1337, scale=1.0):
        import torch

        p = torch.empty(self.n_params, dtype=torch.float32, device="cuda")
        _check(load().tcnnb_encoding_initialize_params(self._h, seed, p.data_ptr(), scale))
        return p

    def fwd(self, x, params16, stream=None):
        import torch

        out = torch.empty(x.shape[0], self.n_output_dims, dtype=torch.float16, device=x.device)
        _check(load().tcnnb_encoding_forward(self._h, _stream_handle(stream), x.shape[0], x.data_ptr(), out.data_ptr(), params16.data_ptr()))
        return out

    def bwd(self, x, params16, dL_doutput, want_params=True, want_input=False, stream=None):
        """-> (dL_dparams fp16 [n_params] or None, dL_dinput fp32 [n][n_input_dims] or None)"""
        import torch

        gp = torch.empty(self.n_params, dtype=torch.float16, device=x.device) if want_params else None
        gx = torch.empty(x.shape[0], self.n_input_dims, dtype=torch.float32, device=x.device) if want_input else None
        _check(load().tcnnb_encoding_backward(self._h, _stream_handle(stream), x.shape[0], gx.data_ptr() if want_input else None, dL_doutput.data_ptr(),
                                              gp.data_ptr() if want_params else None, x.data_ptr(), params16.data_ptr()))
        return gp, gx

    def close(self):
        if self._h:
            load().tcnnb_encoding_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class Network:
    """tcnn::create_network (network.h / cpp_api.h:122): a FullyFusedMLP on its own, caller-owned fp16 parameters."""

    def __init__(self, n_input_dims, n_output_dims, network_config):
        lib = load()
        h = ctypes.c_void_p()
        text = network_config if isinstance(network_config, str) else json.dumps(network_config)
        _check(lib.tcnnb_network_create(n_input_dims, n_output_dims, text.encode(), ctypes.byref(h)))
        self._h = h
        self.n_input_dims, self.n_output_dims = n_input_dims, n_output_dims
        self.n_params = lib.tcnnb_network_n_params(h)
        self.input_width = lib.tcnnb_network_input_width(h)
        self.padded_output_width = lib.tcnnb_network_padded_output_width(h)
        self.width = lib.tcnnb_network_width(h)
        self.n_hidden_layers = lib.tcnnb_network_n_hidden_layers(h)

    def initial_params(self, seed=1337, scale=1.0):
        import torch

        p = torch.empty(self.n_params, dtype=torch.float32, device="cuda")
        _check(load().tcnnb_network_initialize_params(self._h, seed, p.data_ptr(), scale))
        return p

    def inference_mixed_precision(self, x16, params16, stream=None):
        """fp16 [n][n_input_dims] -> fp16 [n][padded_output_width]."""
        import torch

        out = torch.empty(x16.shape[0], self.padded_output_width, dtype=torch.float16, device=x16.device)
        _check(load().tcnnb_network_inference_mixed_precision(self._h, _stream_handle(stream), x16.shape[0], x16.data_ptr(), out.data_ptr(), params16.data_ptr()))
        return out

    def forward(self, x16, params16, stream=None):
        """-> (output fp16 [n][padded_out], hidden fp16 [n_hidden_layers][n][width])"""
        import torch

        n = x16.shape[0]
        out = torch.empty(n, self.padded_output_width, dtype=torch.float16, device=x16.device)
        hidden = torch.empty(self.n_hidden_layers, n, self.width, dtype=torch.float16, device=x16.device)
        _check(load().tcnnb_network_forward(self._h, _stream_handle(stream), n, x16.data_ptr(), out.data_ptr(), hidden.data_ptr(), params16.data_ptr()))
        return out, hidden

    def backward(self, x16, out16, hidden, dL_doutput16, params16, want_input_grad=True, want_param_grad=True, stream=None):
        """Network<T>::backward from the forward pass's input / output / hidden activations:
        -> (dL_dinput fp16 [n][n_input_dims] or None, dL_dparams fp16 [n_params] or None)."""
        import torch

        n = x16.shape[0]
        dx = torch.empty(n, self.input_width, dtype=torch.float16, device=x16.device) if want_input_grad else None
        dp = torch.empty(self.n_params, dtype=torch.float16, device=x16.device) if want_param_grad else None
        _check(load().tcnnb_network_backward(self._h, _stream_handle(stream), n, x16.data_ptr(), out16.data_ptr() if out16 is not None else None, hidden.data_ptr(), dL_doutput16.data_ptr(),
                                             params16.data_ptr(), dx.data_ptr() if dx is not None else None, dp.data_ptr() if dp is not None else None))
        return dx, dp

    def module_inference(self, x32, params16, stream=None):
        """cpp::Module::inference of cpp::create_network: fp32 [n][n_input_dims] (Identity encoding) -> fp16 [n][padded_output_width]."""
        import torch

        out = torch.empty(x32.shape[0], self.padded_output_width, dtype=torch.float16, device=x32.device)
        _check(load().tcnnb_network_module_inference(self._h, _stream_handle(stream), x32.shape[0], x32.data_ptr(), out.data_ptr(), params16.data_ptr()))
        return out

    def module_backward(self, x32, dL_doutput16, params16, want_input_grad=True, want_param_grad=True, stream=None):
        """cpp::Module::backward of cpp::create_network: -> (dL_dinput fp32 [n][n_input_dims] or None, dL_dparams fp16 or None)."""
        import torch

        n = x32.shape[0]
        dx = torch.empty(n, self.n_input_dims, dtype=torch.float32, device=x32.device) if want_input_grad else None
        dp = torch.empty(self.n_params, dtype=torch.float16, device=x32.device) if want_param_grad else None
        _check(load().tcnnb_network_module_backward(self._h, _stream_handle(stream), n, dx.data_ptr() if dx is not None else None, dL_doutput16.data_ptr(),
                                                    dp.data_ptr() if dp is not None else None, x32.data_ptr(), params16.data_ptr()))
        return dx, dp

    def inference(self, x32, params16, stream=None):
        """fp32 [n][n_input_dims] through the Identity encoding -> fp32 [n][n_output_dims]."""
        import torch

        out = torch.empty(x32.shape[0], self.n_output_dims, dtype=torch.float32, device=x32.device)
        _check(load().tcnnb_network_inference(self._h, _stream_handle(stream), x32.shape[0], x32.data_ptr(), out.data_ptr(), params16.data_ptr()))
        return out

    def close(self):
        if self._h:
            load().tcnnb_network_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # noqa: BLE001
            pass


class TrainableModel:
    """Result of create_from_config (config.h:46-51): .network and .trainer share one parameter set."""

    def __init__(self, n_input_dims, n_output_dims, config, seed=1337):
        lib = load()
        handle = ctypes.c_void_p()
        text = config if isinstance(config, str) else json.dumps(config)
        rc = lib.tcnnb_create_from_config(n_input_dims, n_output_dims, text.encode(), seed, ctypes.byref(handle))
        _check(rc)
        self._h = handle
        self.n_input_dims = n_input_dims
        self.n_output_dims = n_output_dims
        self.n_params = lib.tcnnb_n_params(handle)
        self.n_mlp_params = lib.tcnnb_n_mlp_params(handle)
        self.encoded_width = lib.tcnnb_encoded_width(handle)
        self.network = _Network(self)
        self.trainer = _Trainer(self)

    def hyperparams(self):
        return json.loads(load().tcnnb_hyperparams(self._h).decode())

    def grid_levels(self):
        lib = load()
        n = ctypes.c_uint32(0)
        offsets = (ctypes.c_uint32 * 129)()
        scales = (ctypes.c_float * 128)()
        res = (ctypes.c_uint32 * 128)()
        _check(lib.tcnnb_grid_levels(self._h, ctypes.byref(n), offsets, scales, res))
        L = n.value
        return {"n_levels": L, "offsets": list(offsets[: L + 1]), "scales": list(scales[:L]), "resolutions": list(res[:L])}

    def set_debug_taps(self, **tensors):
        taps = DebugTaps()
        for k, t in tensors.items():
            setattr(taps, k, t.data_ptr() if t is not None else None)
        _check(load().tcnnb_set_debug_taps(self._h, ctypes.byref(taps)))

    def set_profiling(self, enable):
        _check(load().tcnnb_set_profiling(self._h, int(enable)))

    def read_profile(self):
        f, o, b, n = ctypes.c_float(0), ctypes.c_float(0), ctypes.c_float(0), ctypes.c_uint32(0)
        _check(load().tcnnb_read_profile(self._h, ctypes.byref(f), ctypes.byref(o), ctypes.byref(b), ctypes.byref(n)))
        return {"fused_ms_total": f.value, "optimizer_ms_total": o.value, "binning_ms_total": b.value, "n_steps": n.value}

    def training_step_host(self, inputs_np, targets_np):
        """C-ABI call with HOST buffers (numpy fp32, C-contiguous): H2D + step + D2H of the loss inside."""
        out = ctypes.c_float(0)
        _check(load().tcnnb_training_step_host(self._h, inputs_np.shape[0], inputs_np.ctypes.data, targets_np.ctypes.data, ctypes.byref(out)))
        return out.value

    def training_step_host_submit(self, inputs_np, targets_np, global_batch=None):
        """Pipelined form: enqueue {H2D, step, D2H of the loss} and return a ticket; up to two steps may be in flight.
        `global_batch` (data-parallel trainer, after dp_init): this call's arrays are the rank's shard of that global batch."""
        t = ctypes.c_uint64(0)
        if global_batch is None:
            _check(load().tcnnb_training_step_host_submit(self._h, inputs_np.shape[0], inputs_np.ctypes.data, targets_np.ctypes.data, ctypes.byref(t)))
        else:
            _check(load().tcnnb_dp_training_step_host_submit(self._h, inputs_np.shape[0], int(global_batch), inputs_np.ctypes.data, targets_np.ctypes.data, ctypes.byref(t)))
        return t.value

    def training_step_host_wait(self, ticket):
        out = ctypes.c_float(0)
        _check(load().tcnnb_training_step_host_wait(self._h, ticket, ctypes.byref(out)))
        return out.value

    def debug_set(self, key, value):
        _check(load().tcnnb_debug_set(self._h, key.encode(), int(value)))

    def inference_host(self, inputs_np, outputs_np):
        _check(load().tcnnb_inference_host(self._h, inputs_np.shape[0], inputs_np.ctypes.data, outputs_np.ctypes.data))
        return outputs_np

    def close(self):
        if self._h:
            load().tcnnb_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def create_from_config(n_input_dims, n_output_dims, config, seed=1337):
    """tcnn::create_from_config (config.h:53-63) + Trainer(..., seed = 1337) (trainer.h:51)."""
    return TrainableModel(n_input_dims, n_output_dims, config, seed)


def kernel_launch_count():
    return load().tcnnb_kernel_launch_count()
