"""GPU: HQQLinear life-cycle -- the reference's own tests/test_quantize.py cases that do not need the HF hub,
plus state_dict interchange with a checkpoint written by the reference."""
import numpy as np
import pytest
import torch

from hqq_b200.core.quantize import BaseQuantizeConfig, HQQBackend, HQQLinear, Quantizer

pytestmark = pytest.mark.gpu
DEV = "cuda"


@pytest.fixture()
def lin():
    torch.manual_seed(42)  # tests/test_quantize.py:22-24
    return torch.nn.Linear(16, 128)


def test_quantizer_float_view_invariance(lin):
    """tests/test_quantize.py:32-48 (default axis=0, gs=64, all bit widths, three compute dtypes)."""
    w = lin.weight.data
    for compute_dtype in [torch.float32, torch.float16, torch.bfloat16]:
        for nbits in [8, 4, 3, 2, 1]:
            W_q, meta = Quantizer.quantize(w, nbits=nbits, round_zero=True, optimize=True, view_as_float=False)
            assert W_q.dtype == (torch.int32 if nbits == 3 else torch.uint8)
            norm1 = torch.norm(w - Quantizer.dequantize(W_q, meta).float(), p=0.7)
            W_q, meta = Quantizer.quantize(w, nbits=nbits, round_zero=True, optimize=True, compute_dtype=compute_dtype, view_as_float=True)
            assert W_q.dtype == compute_dtype
            norm2 = torch.norm(w - Quantizer.dequantize(W_q, meta).float(), p=0.7)
            assert torch.equal(norm1, norm2)


def test_quantizer_cuda_source(lin):
    """tests/test_quantize.py:50-60"""
    w = lin.weight.data.cuda()
    W_q, meta = Quantizer.quantize(w, round_zero=True, optimize=True, view_as_float=False)
    n1 = torch.norm(w - Quantizer.dequantize(W_q, meta), p=0.7)
    W_q, meta = Quantizer.quantize(w, round_zero=True, optimize=True, view_as_float=True)
    n2 = torch.norm(w - Quantizer.dequantize(W_q, meta), p=0.7)
    assert W_q.is_cuda and torch.equal(n1, n2)


def test_floatview_bitpacking():
    """tests/test_quantize.py:62-73 (a subset of its shapes)."""
    for compute_dtype in [torch.float32, torch.float16, torch.bfloat16]:
        for nbits in [8, 4, 3, 2, 1]:
            for shape in [[32, 32], [256, 256], [1024, 1024], [8192, 128], [32, 4096]]:
                pk = Quantizer.bit_to_packing[nbits]
                vd = Quantizer.unpack_view_dtype[pk]
                W = torch.randint(0, 2 ** nbits, shape, device=DEV).to(vd)
                orig = Quantizer.pack[pk](W)
                view = orig.clone().view(compute_dtype)
                assert view.dtype == compute_dtype and torch.equal(orig, view.view(vd))


def test_forward_int_view_vs_float_view(lin):
    """tests/test_quantize.py:123-163 reduced to the non-deprecated options: same outputs whether W_q is stored as
    integers or viewed as compute_dtype, x = [1, 4096, 16], group sizes 8..64 (weight is 128x16)."""
    for compute_dtype in [torch.float32, torch.float16, torch.bfloat16]:
        for nbits in [4, 3, 2]:
            for gs in [8, 16, 32, 64]:
                a = HQQLinear(lin, BaseQuantizeConfig(nbits=nbits, group_size=gs, view_as_float=False), compute_dtype=compute_dtype, del_orig=False)
                b = HQQLinear(lin, BaseQuantizeConfig(nbits=nbits, group_size=gs, view_as_float=True), compute_dtype=compute_dtype, del_orig=False)
                x = torch.randn([1, 4096, 16], device=DEV).to(compute_dtype)
                with torch.no_grad():
                    assert torch.allclose(a.forward(x), b.forward(x), rtol=1e-5)


def test_deprecated_meta_options_are_ignored_like_the_reference(lin):
    cfg = BaseQuantizeConfig(nbits=4, group_size=64, quant_zero=True, quant_scale=True)
    layer = HQQLinear(lin, cfg, compute_dtype=torch.float16, del_orig=False)
    assert layer.quant_config["scale_quant_params"] is None and layer.quant_config["zero_quant_params"] is None
    assert "scale" in layer.meta and "zero" in layer.meta


def test_offload_meta_layout(lin):
    layer = HQQLinear(lin, BaseQuantizeConfig(nbits=4, group_size=64, offload_meta=True), compute_dtype=torch.float16, del_orig=False)
    assert "zero_scale" in layer.meta and not layer.meta["zero_scale"].is_cuda and "scale" not in layer.meta
    plain = HQQLinear(lin, BaseQuantizeConfig(nbits=4, group_size=64), compute_dtype=torch.float16, del_orig=False)
    x = torch.randn(2, 16, device=DEV).half()
    assert torch.allclose(layer(x), plain(x), rtol=1e-3, atol=1e-3)
    assert "scale" not in layer.meta  # temporaries are dropped again (quantize.py:875-877)


def test_state_dict_roundtrip_and_reference_checkpoint(golden):
    torch.manual_seed(0)
    src = torch.nn.Linear(256, 128, bias=True)
    a = HQQLinear(src, BaseQuantizeConfig(nbits=4, group_size=64, axis=1), compute_dtype=torch.float16, device=DEV)
    sd = a.state_dict()
    assert set(sd) == a.state_dict_keys() - set()  # bias present
    assert all(isinstance(v, torch.Tensor) for v in sd.values())  # safetensors-ready
    b = HQQLinear(None, None, compute_dtype=torch.float16, device=DEV, initialize=False)
    b.load_state_dict({k: v.clone() for k, v in sd.items()})
    x = torch.randn(5, 256, device=DEV).half()
    assert torch.equal(a(x), b(x)) and b.in_features == 256 and b.out_features == 128
    assert b.quant_config["weight_quant_params"]["nbits"] == 4 and b.meta["packing"] == "4bit_u8"

    # a state_dict written by the reference itself (64x64 layer, fp32 compute, encoded for safetensors)
    ref_sd = {k[3:]: torch.from_numpy(np.array(golden.state_dict[k])) for k in golden.state_dict.files}
    c = HQQLinear(None, None, compute_dtype=torch.float32, device=DEV, initialize=False)
    c.load_state_dict(ref_sd)
    assert c.meta["nbits"] == 4 and c.meta["shape"] == torch.Size([64, 64]) and c.meta["compute_dtype"] == torch.float32
    assert c.W_q.is_cuda and tuple(c.dequantize().shape) == (64, 64)
    # and our encoding of the same layer is tensor-for-tensor what the reference wrote
    out = c.state_dict()
    for k, v in out.items():
        if k in ("W_q", "scale", "zero", "bias"):
            continue
        assert torch.equal(v.cpu(), torch.from_numpy(np.array(golden.state_dict["sd/" + k]))), k


def test_module_plumbing(lin):
    m = torch.nn.Sequential(HQQLinear(lin, BaseQuantizeConfig(nbits=4, group_size=64), compute_dtype=torch.float16, del_orig=False))
    assert m.half() is m and m[0].W_q.dtype == torch.uint8  # casts are no-ops on quantised layers
    full = m.state_dict()
    assert "0.W_q" in full and "0.nbits" in full
    m2 = torch.nn.Sequential(HQQLinear(None, None, compute_dtype=torch.float16, device=DEV, initialize=False))
    m2.load_state_dict(full)
    x = torch.randn(2, 16, device=DEV).half()
    assert torch.equal(m(x), m2(x))
    assert "in_features=16, out_features=128" in repr(m2[0])


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_layers_on_a_device_that_is_not_current():
    """BaseHQQModel.quantize_model(device=[...]) spreads layers over GPUs of one process: a layer on cuda:1 must launch on cuda:1 while
    cuda:0 is current (the C ABI launches on the calling thread's current device: ops.py guards it, the function-attribute and grid
    caches of the kernels are per device) -- every route: one-token kernel, small-M kernel, wgmma GEMM, dequantize + dense GEMM."""
    torch.manual_seed(21)
    assert torch.cuda.current_device() == 0
    for cfg in (dict(nbits=4, group_size=64, axis=1), dict(nbits=3, group_size=64, axis=1)):
        lin = torch.nn.Linear(2048, 1024, bias=True)
        W, b = lin.weight.data.clone(), lin.bias.data.clone()
        layers = [HQQLinear.from_weights(W.clone().half(), torch.nn.Parameter(b.clone().half()), BaseQuantizeConfig(**cfg), compute_dtype=torch.float16,
                                         device=d) for d in ("cuda:0", "cuda:1")]
        for M in (1, 8, 300):
            x = torch.randn(M, 2048).half()
            y0 = layers[0](x.to("cuda:0"))
            y1 = layers[1](x.to("cuda:1"))
            assert y1.device.index == 1
            assert torch.equal(y0.cpu(), y1.cpu()), (cfg, M)
    assert torch.cuda.current_device() == 0
