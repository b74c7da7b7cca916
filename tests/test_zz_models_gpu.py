"""GPU: the model walker end to end (SURVEY.md 8 f-1) -- a tiny Llama is quantised through `AutoHQQHFModel.quantize_model` on the
GPU and compared with the checkpoint the REAL reference produced from the same dense weights (tests/golden/models)."""
import os

import pytest
import torch

from hqq_b200.core.quantize import BaseQuantizeConfig, HQQLinear
from hqq_b200.models.hf.base import AutoHQQHFModel

pytestmark = pytest.mark.gpu
transformers = pytest.importorskip("transformers")
GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "models")


# Written after round 1's GPU budget was spent: the first execution is the driver's round-end run.  Non-strict, so it reports
# XPASS when it holds; the mark goes away once it has been seen green.
def test_quantize_model_matches_the_reference_checkpoint(tmp_path):
    dev = "cuda:0"
    cfg = transformers.AutoConfig.from_pretrained(os.path.join(GOLD, "quantized", "config.json"))
    model = transformers.LlamaForCausalLM(cfg)
    model.load_state_dict(torch.load(os.path.join(GOLD, "dense_state_dict.pt"), weights_only=True))
    quant_config = {"self_attn.q_proj": BaseQuantizeConfig(nbits=4, group_size=64, axis=1),
                    "self_attn.k_proj": BaseQuantizeConfig(nbits=4, group_size=64, axis=1),
                    "self_attn.v_proj": BaseQuantizeConfig(nbits=8, group_size=64, axis=1),
                    "self_attn.o_proj": None,
                    "mlp.gate_proj": BaseQuantizeConfig(nbits=2, group_size=64, axis=1),
                    "mlp.up_proj": BaseQuantizeConfig(nbits=3, group_size=64, axis=1),
                    "mlp.down_proj": BaseQuantizeConfig(nbits=4, group_size=64, axis=0)}
    AutoHQQHFModel.quantize_model(model, quant_config, compute_dtype=torch.float32, device=dev)
    ref = AutoHQQHFModel.from_quantized(os.path.join(GOLD, "quantized"), compute_dtype=torch.float32, device=dev, cache_dir=None)
    n = 0
    for (name, ours), (_, theirs) in zip(model.named_modules(), ref.named_modules()):
        assert type(ours).__name__ == type(theirs).__name__, name
        if isinstance(ours, HQQLinear):
            n += 1
            assert ours.meta["nbits"] == theirs.meta["nbits"] and ours.meta["axis"] == theirs.meta["axis"] and ours.W_q.shape == theirs.W_q.shape
            Wa, Wb = ours.dequantize().float(), theirs.dequantize().float()
            step = theirs.meta["scale"].float().abs().max()
            # the on-chip solver may flip a half-way tie (one level, and that group's zero moves by 1/gs of a level)
            assert (Wa - Wb).abs().max() <= 1.1 * step, name
            assert ((Wa - Wb).abs() > 0.05 * step).float().mean() <= 1e-2, name
        elif isinstance(ours, torch.nn.Linear):
            assert torch.equal(ours.weight, theirs.weight), name
    assert n == 4 * 6
    ids = torch.arange(12, device=dev).view(1, 12) % cfg.vocab_size
    with torch.no_grad():
        la, lb = model(ids).logits.float(), ref(ids).logits.float()
    assert torch.isfinite(la).all()
    assert (la - lb).norm() / lb.norm() <= 2e-2
    # save with our writer, load with our reader: identical logits
    out = str(tmp_path / "q")
    AutoHQQHFModel.save_quantized(model, out)
    again = AutoHQQHFModel.from_quantized(out, compute_dtype=torch.float32, device=dev, cache_dir=None)
    with torch.no_grad():
        assert torch.equal(again(ids).logits.float(), la)


def test_batched_decode_matches_single_sequences():
    """DecodeModel(batch=3): the fused small-M kernel (M = 3) between framework glue ops, captured in a CUDA graph; every sequence
    decodes the tokens it decodes alone (batch = 1, same unfused path).  Near-ties may flip late tokens: the first ones must agree."""
    from hqq_b200 import harness
    dev = torch.device("cuda", 0)
    shape = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
    first = [5, 9, 11]

    def run(batch, toks):
        m = harness.DecodeModel(shape, dtype=torch.float16, device=dev, cache_len=32, fused=False, seed=3, batch=batch)
        m.capture()
        m.tok.copy_(torch.tensor(toks, device=dev)); m.pos.zero_()
        for blk in m.blocks:
            blk["k_cache"].zero_(); blk["v_cache"].zero_()
        out = []
        for _ in range(8):
            m.decode()
            out.append(m.next_tok.clone())
        return torch.stack(out, 1).cpu()

    together = run(3, first)
    for i, t in enumerate(first):
        alone = run(1, [t])[0]
        assert torch.equal(together[i][:3], alone[:3]), (i, together[i], alone)
        assert int((together[i] == alone).sum()) >= 6, (i, together[i], alone)
