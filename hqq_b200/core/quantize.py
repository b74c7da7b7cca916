"""Drop-in surface of ``hqq.core.quantize`` -- ``Quantizer``, ``HQQLinear``, ``HQQBackend``,
``BaseQuantizeConfig`` -- backed by ONE sm_90a code path (``libhqq_b200.so``).

What maps to what (reference: mobiusml/hqq @ e0b1d00, hqq/core/quantize.py):
  Quantizer.quantize          :76-180   -> hqq_b200_quantize (fused min/max init + proximal solver + pack)
  Quantizer.dequantize        :184-199  -> hqq_b200_dequantize (both axes, all bit widths)
  HQQLinear.forward (any HQQBackend member, :269-285,:888-1052)
                                         -> hqq_b200_linear_fwd (fused unpack->dequant->MMA); configurations the
                                            fused kernels do not cover run hqq_b200_dequantize + torch.matmul
  HQQLinear.state_dict / load_state_dict :617-787 -> same keys and tensor encodings (safetensors compatible)
There is no Triton, no torch.compile, no per-backend dispatch and no CPU arithmetic: ``HQQBackend`` keeps its
members so callers' ``set_backend`` lines keep working, but every member resolves to the same kernels.
"""
from __future__ import annotations

import copy
from enum import Enum
from typing import Union

import torch
from torch import Tensor, bfloat16, float16, int32, nn, uint8

from .. import ops
from .bitpack import BitPack
from .optimize import optimize_weights_proximal
from .utils import decode_safetensor_type, encode_safetensor_type, is_divisible

_META_TYPE = {
    "scale": torch.Tensor, "zero": torch.Tensor, "zero_scale": torch.Tensor,
    "compute_dtype": torch.dtype, "quant_zero": bool, "quant_scale": bool, "view_as_float": bool,
    "unpack_view_dtype": torch.dtype, "packing": str, "axis": int, "group_size": int, "nbits": int,
    "shape": torch.Size, "channel_wise": bool, "optimize": bool, "round_zero": bool,
}

_FUSED_BITS = (8, 4, 3, 2, 1)  # bit widths with a real packing (and kernels); 6/5/1.58 are stored as 8/8/2-bit


def _warn(msg: str) -> None:
    print(msg)


def _cuda_device(device) -> torch.device:
    dev = torch.device(device) if device is not None else torch.device("cuda")
    if dev.type != "cuda":
        if not torch.cuda.is_available():
            raise RuntimeError("hqq_b200: a CUDA device (H100, sm_90a) is required; there is no CPU path")
        dev = torch.device("cuda", torch.cuda.current_device())
    if dev.index is None:
        dev = torch.device("cuda", torch.cuda.current_device())
    return dev


class Quantizer:
    SUPPORTED_BITS = [8, 6, 5, 4, 3, 2, 1.58, 1]
    optimize_weights = optimize_weights_proximal  # the solver seam; replaceable exactly like the reference's

    bit_to_packing = {8: "8bit_u8", 6: "8bit_u8", 5: "8bit_u8", 4: "4bit_u8", 3: "3bit_32", 2: "2bit_u8",
                      1.58: "2bit_u8", 1: "1bit_u8"}
    pack = {"8bit_u8": BitPack.pack_8bit_u8, "4bit_u8": BitPack.pack_4bit_u8, "3bit_32": BitPack.pack_3bit_32,
            "2bit_u8": BitPack.pack_2bit_u8, "1bit_u8": BitPack.pack_1bit_u8}
    unpack = {"8bit_u8": BitPack.unpack_8bit_u8, "4bit_u8": BitPack.unpack_4bit_u8, "3bit_32": BitPack.unpack_3bit_32,
              "2bit_u8": BitPack.unpack_2bit_u8, "1bit_u8": BitPack.unpack_1bit_u8}
    unpack_view_dtype = {"8bit_u8": uint8, "4bit_u8": uint8, "3bit_32": int32, "2bit_u8": uint8, "1bit_u8": uint8}
    _packing_bits = {"8bit_u8": 8, "4bit_u8": 4, "3bit_32": 3, "2bit_u8": 2, "1bit_u8": 1}

    @classmethod
    def quantize(cls, tensor: Tensor, nbits: float = 4, channel_wise: bool = True, group_size: int = 64,
                 optimize: bool = True, round_zero: bool = False, axis: int = 0, bitpack: bool = True,
                 compute_dtype: Union[torch.dtype, None] = None, view_as_float: bool = False, device: str = "cuda") -> tuple:
        assert nbits in Quantizer.SUPPORTED_BITS, "nbits=" + str(nbits) + " not supported."
        assert axis in [0, 1], "axis should be either 0 or 1"
        if group_size is not None:
            assert is_divisible(tensor.numel(), group_size), (
                "group_size should be divisble by the total tensor dimensions. shape: "
                + str(tensor.shape) + ", group_size: " + str(group_size))

        home = tensor.device
        dev = tensor.device if tensor.is_cuda else _cuda_device(device)
        shape = tensor.shape
        W = tensor.to(dev)
        if W.dtype not in (torch.float32, torch.float16, torch.bfloat16):
            W = W.float()
        W2d = W.reshape(shape[0], -1) if W.dim() != 2 else W
        packing = Quantizer.bit_to_packing[nbits]
        store_bits = Quantizer._packing_bits[packing]
        max_v = round(2 ** nbits - 1)

        fused = (channel_wise and group_size is not None and bitpack
                 and cls.optimize_weights is optimize_weights_proximal)
        if fused:
            # hot path (a): one C call = min/max init + 20-iteration proximal solver + round/clamp + slab packing
            W_q, scale, zero, _ = ops.quantize(W2d, nbits=store_bits, group_size=group_size, axis=axis,
                                               round_zero=round_zero, optimize=optimize, max_level=max_v)
            meta_shape = (-1, 1) if axis == 1 else (1, -1)
            scale, zero = scale.reshape(meta_shape), zero.reshape(meta_shape)
        else:
            W_q, scale, zero = cls._quantize_seam(W2d.float(), nbits, channel_wise, group_size, optimize, round_zero, axis, dev)
            if bitpack:
                W_q = Quantizer.pack[packing](W_q)
            else:
                W_q = W_q.to(tensor.dtype)

        meta = {"nbits": nbits, "group_size": group_size, "shape": shape, "scale": scale.to(home), "zero": zero.to(home),
                "axis": axis, "packing": packing if bitpack else None}
        meta["unpack_view_dtype"] = Quantizer.unpack_view_dtype[packing]
        meta["view_as_float"] = view_as_float
        if bitpack and view_as_float:
            W_q = W_q.view(torch.float32 if compute_dtype is None else compute_dtype)
        return W_q.to(home), meta

    @classmethod
    def _quantize_seam(cls, W, nbits, channel_wise, group_size, optimize, round_zero, axis, dev):
        """Generic route (custom ``Quantizer.optimize_weights``, ``channel_wise=False`` or ``bitpack=False``):
        the reference's steps quantize.py:104-149 as device tensor ops around the solver seam."""
        if group_size is not None and channel_wise:
            W = W.reshape([-1, group_size]) if axis == 1 else W.reshape([group_size, -1])
        if not channel_wise:
            _min, _max = W.min(), W.max()
            optimize = False
        else:
            _min = W.min(axis=axis, keepdim=True)[0]
            _max = W.max(axis=axis, keepdim=True)[0]
        max_v = round(2 ** nbits - 1)
        denom = _max - _min
        scale = max_v / denom
        scale = torch.where(denom.abs() <= 1e-4, torch.full_like(scale, 1.0), scale).clamp(max=2e4)
        zero = -_min * scale
        if round_zero:
            zero = torch.round(zero)
        if optimize:
            W_q, scale, zero = cls.optimize_weights(tensor=W, scale=scale, zero=zero, min_max=[0, max_v], axis=axis, device=str(dev))
        else:
            W_q = (W * scale + zero).round_().clamp_(0, max_v)
        return W_q, 1.0 / scale, zero

    # Main dequantization: bit_unpacking > (W_q - z)*s > reshape            (quantize.py:184-199)
    @classmethod
    def dequantize(cls, W_q: Tensor, meta: dict) -> Tensor:
        compute_dtype = meta["compute_dtype"] if ("compute_dtype" in meta) else float16
        if meta["packing"]:
            if meta["view_as_float"]:
                W_q = W_q.view(meta["unpack_view_dtype"])
            shape = meta["shape"]
            gs = meta["group_size"]
            if gs is not None and len(shape) == 2 and meta["scale"].numel() * gs == shape[0] * shape[1]:
                return ops.dequantize(W_q, meta["scale"], meta["zero"], shape, gs, Quantizer._packing_bits[meta["packing"]],
                                      meta["axis"], compute_dtype)
            # scalar meta (channel_wise=False) or unusual shapes: unpack with the kernel, affine map with tensor ops
            W_r = Quantizer.unpack[meta["packing"]](W_q, dtype=compute_dtype)
            if meta["nbits"] == 3:
                rows = gs if meta["axis"] == 0 else (shape[0] * shape[1] // gs)
                W_r = W_r[:rows]
        else:
            W_r = W_q.to(compute_dtype)
        return ((W_r - meta["zero"]) * meta["scale"]).reshape(meta["shape"])

    @classmethod
    def to_inplace(cls, W_q: Tensor, meta: dict, device) -> tuple:
        compute_dtype = meta["compute_dtype"] if ("compute_dtype" in meta) else float16
        if W_q is not None:
            W_q = W_q.to(device).contiguous()
        for key in meta:
            if isinstance(meta[key], torch.Tensor):
                t = meta[key]
                meta[key] = (t.to(compute_dtype) if torch.is_floating_point(t) else t).to(device).contiguous()
        return W_q, meta

    @classmethod
    def to_ooplace(cls, W_q: Tensor, meta: dict, device) -> tuple:
        compute_dtype = meta["compute_dtype"] if ("compute_dtype" in meta) else float16
        W_q_c = W_q.to(device).contiguous() if W_q is not None else None
        meta_c = {}
        for key, t in meta.items():
            if isinstance(t, torch.Tensor):
                meta_c[key] = (t.to(compute_dtype) if torch.is_floating_point(t) else t).to(device).contiguous()
            else:
                meta_c[key] = t
        return W_q_c, meta_c

    @classmethod
    def cuda(cls, W_q: Tensor, meta: dict, device) -> tuple:
        return Quantizer.to_inplace(W_q, meta, device=device)

    @classmethod
    def cpu(cls, W_q: Tensor, meta: dict) -> tuple:
        return Quantizer.to_ooplace(W_q, meta, device="cpu")


class HQQBackend(Enum):
    # Same members / values as the reference (quantize.py:269-285): the value is the name of the forward method.
    PYTORCH = "forward_pytorch_backprop"
    PYTORCH_COMPILE = "forward_pytorch_backprop_compile"
    ATEN = "forward_aten_backprop"
    PYTORCH_BACKPROP = "forward_pytorch_backprop"
    PYTORCH_BACKPROP_COMPILE = "forward_pytorch_backprop_compile"
    ATEN_BACKPROP = "forward_aten_backprop"
    PYTORCH_FORWARD = "forward_pytorch"
    PYTORCH_FORWARD_COMPILE = "forward_pytorch_compile"
    ATEN_FORWARD = "forward_aten"
    ATEN_FORWARD_INT8 = "forward_aten_int8"


class HQQMatmulNoCacheMul(torch.autograd.Function):
    """y = x @ W_r^T (+ bias) with the fused kernel in forward; grad_input = grad @ W_r in backward
    (quantize.py:322-352).  The quantised weight itself has no gradient."""

    @staticmethod
    def forward(x, layer, bias):
        return layer._fused_forward(x)

    @staticmethod
    def setup_context(ctx, inputs, outputs):
        x, layer, bias = inputs
        ctx.save_for_backward(x, bias)
        ctx.layer = layer

    @staticmethod
    def backward(ctx, grad_output):
        x, bias = ctx.saved_tensors
        grad_input = grad_bias = None
        if ctx.needs_input_grad[0]:
            grad_input = ctx.layer.matmul(grad_output, transpose=False)  # grad @ W_r on the dense wgmma kernel (W_r^T as the weight)
        if bias is not None and ctx.needs_input_grad[2]:
            grad_bias = grad_output.reshape(-1, grad_output.shape[-1]).sum(0)
        return grad_input, None, grad_bias


# Main linear layer
class HQQLinear(nn.Module):
    backend = HQQBackend.PYTORCH

    def __init__(self, linear_layer: Union[nn.Module, None], quant_config: dict, del_orig: bool = True,
                 compute_dtype: torch.dtype = float16, device: str = "cuda", initialize: bool = True):
        super().__init__()
        self.ready = False
        self.in_gpu = False
        self.bias = None
        self.axis = None
        self.channel_wise = None
        self.device = device
        self.compute_dtype = compute_dtype
        self.quant_config = copy.deepcopy(quant_config)
        self.del_orig = del_orig
        self.offload_meta = self.quant_config.pop("offload_meta") if (self.quant_config is not None) else None
        self.set_backend(HQQLinear.backend)
        self.linear_layer = linear_layer
        self.W_q = None
        self.meta = None
        self.encoded_state_dict = True  # state_dict values are tensors -> safetensors compatible
        if initialize:
            self.initialize()

    def is_initialized(self):
        return self.W_q is not None and self.meta is not None

    def initialize(self):
        if self.linear_layer is None:
            return
        qc = self.quant_config
        if qc["scale_quant_params"] is not None or qc["zero_quant_params"] is not None:
            _warn("Warning: Quantizing zeros/scales is deprecated. This setting will be ignored.")
            qc["scale_quant_params"] = None
            qc["zero_quant_params"] = None
        wq = qc["weight_quant_params"]
        if wq["group_size"] is None:  # whole row / column as one group (quantize.py:442-447)
            wq["group_size"] = self.linear_layer.in_features if wq["axis"] == 1 else self.linear_layer.out_features
        self.quantize(self.linear_layer.weight.data, **qc)
        b = self.linear_layer.bias
        self.bias = None if b is None else b.clone().to(device=self.device, dtype=self.compute_dtype)
        if self.del_orig:
            for name, _ in list(self.linear_layer.named_parameters()):
                setattr(self.linear_layer, name, None)
            del self.linear_layer
            torch.cuda.empty_cache()

    @classmethod
    def from_weights(cls, weight: Tensor, bias: Union[Tensor, None], quant_config: dict, compute_dtype: torch.dtype = float16,
                     device: str = "cuda", del_orig: bool = True):
        dummy = torch.nn.Linear(1, 1)
        dummy.in_features, dummy.out_features = weight.shape[1], weight.shape[0]
        dummy.weight.data = weight
        # the reference assigns `bias` as is (quantize.py:826), which nn.Module only accepts for None / nn.Parameter; a plain tensor is
        # wrapped here instead of raising
        dummy.bias = bias if (bias is None or isinstance(bias, nn.Parameter)) else nn.Parameter(bias, requires_grad=False)
        return cls(dummy, quant_config=quant_config, compute_dtype=compute_dtype, device=device, del_orig=del_orig)

    def extra_repr(self) -> str:
        if getattr(self, "meta", None) is not None:
            in_features, out_features = self.meta["shape"][::-1]
            return f"in_features={in_features}, out_features={out_features}, bias={self.bias is not None}"
        return ""

    @classmethod
    def set_backend(cls, backend: HQQBackend):
        # All members lead to the same sm_90a kernels; the attribute is kept for API compatibility.
        HQQLinear.backend = backend
        cls.forward = getattr(cls, backend.value)

    # ------------------------------------------------------------------ device placement (quantize.py:515-583)
    def cuda(self, device):
        self.meta["compute_dtype"] = self.compute_dtype
        if isinstance(self.W_q, nn.parameter.Parameter):
            self.W_q.data, self.meta = Quantizer.cuda(self.W_q.data, self.meta, device)
        else:
            self.W_q, self.meta = Quantizer.cuda(self.W_q, self.meta, device)
        for flag, qk, mk, plain in (("quant_zero", "zero_q", "meta_zero", "zero"), ("quant_scale", "scale_q", "meta_scale", "scale")):
            if self.meta.get(flag, False):
                if qk in self.meta:
                    self.meta[qk], self.meta[mk] = Quantizer.cuda(self.meta[qk], self.meta[mk], device)
                else:
                    _, self.meta[mk] = Quantizer.cuda(None, self.meta[mk], device)
            elif plain in self.meta:
                self.meta[plain] = self.meta[plain].to(device)
        if self.offload_meta:
            if "zero_scale" not in self.meta:
                if self.meta.get("quant_scale") and self.meta.get("quant_zero"):
                    self.meta["zero_scale"] = torch.stack((self.meta["zero_q"], self.meta["scale_q"]))
                    del self.meta["scale_q"], self.meta["zero_q"]
                else:
                    self.meta["zero_scale"] = torch.stack((self.meta["zero"], self.meta["scale"])).to(self.compute_dtype)
                    del self.meta["scale"], self.meta["zero"]
            self.meta["zero_scale"] = self.meta["zero_scale"].contiguous().cpu().pin_memory()
        if self.bias is not None:
            if isinstance(self.bias, torch.nn.Parameter):
                self.bias.data = self.bias.data.to(device=device, dtype=self.compute_dtype)
            elif isinstance(self.bias, torch.Tensor):
                self.bias = self.bias.to(device=device, dtype=self.compute_dtype)
        self.W_q = nn.Parameter(self.W_q, requires_grad=False)
        self.device = device
        self.in_gpu = True
        return self

    # dtype / device casts are no-ops on a quantised layer, as in the reference (quantize.py:585-611)
    def to(self, *args, **kwargs):
        return self

    def type(self, dst_type):
        return self

    def half(self, *args, **kwargs):
        return self

    def bfloat16(self, *args, **kwargs):
        return self

    def float(self, *args, **kwargs):
        return self

    def double(self, *args, **kwargs):
        return self

    def cpu(self):
        return self

    # ------------------------------------------------------------------ state_dict codec (quantize.py:617-787)
    def state_dict_keys(self):
        return {"W_q", "nbits", "group_size", "shape", "scale", "zero", "axis", "packing", "unpack_view_dtype",
                "view_as_float", "quant_scale", "quant_zero", "compute_dtype", "bias", "offload_meta",
                "encoded_state_dict", "stores_quant_config", "channel_wise", "optimize", "round_zero"}

    def state_dict(self, *args, **kwargs):  # nn.Module override compatible
        if not self.is_initialized():
            return {k: None for k in self.state_dict_keys()}
        if (self.quant_config["scale_quant_params"] or self.quant_config["zero_quant_params"]) and self.encoded_state_dict:
            raise Exception("Unsupported serialization for quantized scale/zero and self.encoded_state_dict=True")
        enc = encode_safetensor_type if self.encoded_state_dict else (lambda z: z)
        state = {"W_q": self.W_q}
        state.update({k: enc(v) for k, v in self.meta.items()})
        if self.bias is not None:
            state["bias"] = self.bias
        state["offload_meta"] = enc(self.offload_meta)
        if self.encoded_state_dict:
            state["encoded_state_dict"] = enc(self.encoded_state_dict)
        state["stores_quant_config"] = enc(True)
        for k, v in self.quant_config["weight_quant_params"].items():
            state[k] = enc(v)
        if "destination" in kwargs and "prefix" in kwargs:
            for key, value in state.items():
                kwargs["destination"][kwargs["prefix"] + key] = value
        return state

    def _load_from_state_dict(self, state_dict, prefix, local_metadata, strict, missing_keys, unexpected_keys, error_msgs):
        layer_sd = {}
        for key in self.state_dict_keys():
            if prefix + key in state_dict:
                layer_sd[key] = state_dict.pop(prefix + key)
            elif key not in ["bias"]:
                missing_keys.append(prefix + key)
        if "W_q" in layer_sd:
            layer_sd["W_q"] = nn.Parameter(layer_sd["W_q"], requires_grad=False)
            self.load_state_dict(layer_sd, strict=strict)
        else:
            missing_keys.append(prefix + "W_q")

    def load_state_dict(self, state_dict, strict=True, assign=False):
        encoded = "encoded_state_dict" in state_dict
        if encoded:
            state_dict.pop("encoded_state_dict")
        dec = decode_safetensor_type if encoded else (lambda z, w: z)
        if state_dict.pop("stores_quant_config", False):
            self.quant_config = {"weight_quant_params": {
                k: dec(state_dict[k], _META_TYPE[k])
                for k in ["nbits", "channel_wise", "group_size", "optimize", "round_zero", "axis", "view_as_float"]}}
            self.quant_config["scale_quant_params"] = state_dict.pop("scale_quant_params", None)
            self.quant_config["zero_quant_params"] = state_dict.pop("zero_quant_params", None)
        self.W_q = state_dict.pop("W_q")
        self.bias = state_dict.pop("bias", None)
        self.offload_meta = dec(state_dict.pop("offload_meta", False), bool)
        if "meta" in state_dict:
            self.meta = state_dict["meta"]  # pre-safetensors checkpoints
        else:
            self.meta = {k: dec(v, _META_TYPE[k]) for k, v in state_dict.items()}
        if self.offload_meta is None:
            self.offload_meta = False
        for key in ["zero", "zero_q", "scale", "scale_q", "zero_scale"]:
            if key in self.meta and self.offload_meta:
                self.meta[key] = self.meta[key].cpu().contiguous().pin_memory()
        self.meta.setdefault("unpack_view_dtype", Quantizer.unpack_view_dtype[self.meta["packing"]])
        self.meta.setdefault("view_as_float", False)
        for mk in ("meta_scale", "meta_zero"):
            if mk in self.meta:
                self.meta[mk].setdefault("view_as_float", False)
        self.meta.setdefault("quant_scale", False)
        self.meta.setdefault("quant_zero", False)
        self.cuda(self.device)
        self.ready = True
        self.in_features, self.out_features = self.meta["shape"][::-1]

    # ------------------------------------------------------------------ quantize (quantize.py:789-833)
    def quantize(self, W: Tensor, weight_quant_params: dict, scale_quant_params: dict, zero_quant_params: dict) -> None:
        quant_scale = scale_quant_params is not None
        quant_zero = zero_quant_params is not None
        self.in_features, self.out_features = W.t().shape
        dev = _cuda_device(self.device)
        # The weight goes to the GPU once; everything up to the packed W_q happens there.
        W_q, meta = Quantizer.quantize(W.to(dev), device=self.device, compute_dtype=self.compute_dtype, **weight_quant_params)
        meta.update({"quant_scale": quant_scale, "quant_zero": quant_zero})
        if quant_zero:
            meta["zero_q"], meta["meta_zero"] = Quantizer.quantize(meta["zero"], device=self.device, view_as_float=False, **zero_quant_params)
            del meta["zero"]
            meta["meta_zero"]["compute_dtype"] = self.compute_dtype
        if quant_scale:
            meta["scale_q"], meta["meta_scale"] = Quantizer.quantize(meta["scale"], device=self.device, view_as_float=False, **scale_quant_params)
            del meta["scale"]
            meta["meta_scale"]["compute_dtype"] = self.compute_dtype
        self.W_q = W_q
        self.meta = meta
        self.cuda(self.device)
        self.ready = True

    def unpack(self, reshape=False, dtype=None):
        if self.ready is False:
            return None
        if self.meta["packing"]:
            W_q = self.W_q.view(self.meta["unpack_view_dtype"]) if self.meta["view_as_float"] else self.W_q
            W_r = Quantizer.unpack[self.meta["packing"]](W_q, dtype=dtype if (dtype is not None) else self.compute_dtype)
            return W_r.view(self.meta["shape"]) if reshape else W_r

    def _resolved_meta(self):
        """meta with plain `scale` / `zero` tensors on the weight's device (resolves the deprecated
        offload / quantised-meta layouts the same way quantize.py:844-878 does), plus the keys to drop after."""
        meta, device = self.meta, self.W_q.device
        drop = set()
        if "zero_scale" in meta:
            zs = meta["zero_scale"].to(device=device)
            if zs.dtype == uint8:
                meta["zero_q"], meta["scale_q"] = zs[0], zs[1]
                drop.update({"zero_q", "scale_q"})
            else:
                meta["zero"], meta["scale"] = zs[0], zs[1]
                drop.update({"zero", "scale"})
        if meta.get("quant_zero", False):
            meta["zero"] = Quantizer.dequantize(meta["zero_q"].to(device=device), meta["meta_zero"])
            drop.add("zero")
        if meta.get("quant_scale", False):
            meta["scale"] = Quantizer.dequantize(meta["scale_q"].to(device=device), meta["meta_scale"])
            drop.add("scale")
        return meta, drop

    def dequantize(self):
        assert self.ready, "model was not quantized"
        meta, drop = self._resolved_meta()
        W_est = Quantizer.dequantize(self.W_q, meta)
        for key in drop:
            del meta[key]
        return W_est

    def matmul(self, x: Tensor, transpose: bool = True) -> Tensor:
        if transpose:
            return self._fused_forward(x, with_bias=False)
        # x @ W_r (the backward of the forward, quantize.py:322-352): the dense wgmma GEMM on W_r^T -- K and N swap roles
        W_r = self.dequantize()
        if x.is_cuda and x.dtype in (float16, bfloat16) and W_r.dtype == x.dtype:
            out = ops.dense_gemm(x.reshape(-1, W_r.shape[0]), W_r.t().contiguous())
            if out is not None:
                return out.reshape(*x.shape[:-1], W_r.shape[1])
        return torch.matmul(x, W_r)

    # ------------------------------------------------------------------ the one forward path
    def _fused_forward(self, x: Tensor, with_bias: bool = True) -> Tensor:
        assert self.ready, "model was not quantized"
        meta = self.meta
        N, K = meta["shape"]
        bias = self.bias if with_bias else None
        gs = meta["group_size"]
        nbits = Quantizer._packing_bits.get(meta["packing"], 0)  # storage width (6/5-bit live in bytes, 1.58 in 2 bits)
        if (x.is_cuda and x.dtype == self.compute_dtype and nbits in _FUSED_BITS and gs is not None
                and "scale" in meta and "zero" in meta and not meta.get("quant_scale") and not meta.get("quant_zero")):
            x2d = x.reshape(-1, K)
            if not x2d.is_contiguous():
                x2d = x2d.contiguous()
            y = ops.linear_fwd(x2d, self.W_q, meta["scale"], meta["zero"], bias, N, K, gs, int(nbits), meta["axis"])
            if y is not None:
                return y.reshape(*x.shape[:-1], N)
        # what no route of hqq_b200_linear_fwd covers (float32 compute, quantised meta): our dequantize kernel, then the dense
        # wgmma GEMM when the compute dtype allows it; float32 has no tensor-core path here and goes to the library GEMM
        W_r = self.dequantize()
        x2d = x.reshape(-1, K)
        out = ops.dense_gemm(x2d, W_r.to(x.dtype), bias) if (x.is_cuda and x.dtype in (float16, bfloat16)) else None
        if out is not None:
            return out.reshape(*x.shape[:-1], N)
        out = torch.matmul(x, W_r.t())
        if bias is not None:
            out += bias
        return out

    def forward_pytorch_backprop(self, x: Tensor) -> Tensor:
        if torch.is_grad_enabled() and x.requires_grad:
            return HQQMatmulNoCacheMul.apply(x, self, self.bias)
        return self._fused_forward(x)

    def forward_pytorch(self, x: Tensor) -> Tensor:
        return self._fused_forward(x)

    # The remaining backend names resolve to the same kernels (north star: one sm_90a path behind HQQBackend).
    forward_pytorch_backprop_compile = forward_pytorch_backprop
    forward_pytorch_compile = forward_pytorch
    forward_aten_backprop = forward_pytorch_backprop
    forward_aten = forward_pytorch
    forward_aten_int8 = forward_pytorch
    forward = forward_pytorch_backprop

    def dequantize_aten(self):
        return self.dequantize()


def hqq_base_quant_config(nbits: int = 4, group_size: int = 64, quant_zero: bool = False, quant_scale: bool = False,
                          offload_meta: bool = False, view_as_float: bool = False, axis: int = 1):
    """Same dictionary as the reference builds (quantize.py:1076-1151), including ``round_zero = (nbits == 4)``."""
    assert nbits in Quantizer.SUPPORTED_BITS, "nbits value not supported. Check Quantizer.SUPPORTED_BITS."
    if group_size is not None:
        assert is_divisible(group_size, 8), "Invalid group_size param: the value should be a multiple of 8."
    weight_quant_params = {"nbits": nbits, "channel_wise": True, "group_size": group_size, "optimize": True,
                           "round_zero": True if nbits == 4 else False, "axis": axis, "view_as_float": view_as_float}
    if quant_zero or quant_scale:
        _warn("Warning: Quantized meta-data is deprecated and will be removed. It is not supported for quantized model serialization.")
    if offload_meta:
        _warn("Warning: Meta-data offloading is deprecated and will be removed. It is not supported for quantized model serialization.")
        if quant_scale != quant_zero:
            quant_scale = quant_zero
    grouped8 = {"nbits": 8, "channel_wise": True, "group_size": 128, "optimize": False}
    scale_quant_params = dict(grouped8) if quant_scale else None
    if offload_meta:
        zero_quant_params = dict(grouped8) if quant_zero else None
    else:
        zero_quant_params = {"nbits": 8, "channel_wise": False, "group_size": None, "optimize": False} if quant_zero else None
    return {"weight_quant_params": weight_quant_params, "scale_quant_params": scale_quant_params,
            "zero_quant_params": zero_quant_params, "offload_meta": offload_meta}


# Alias: follow similar Auto-GPTQ naming
BaseQuantizeConfig = hqq_base_quant_config
