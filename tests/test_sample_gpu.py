"""hqq_b200_glue_sample on the H100 and the decode harness with do_sample.

Kernel tokens are held to tests/sample_ref.py's rule against the float64 restatement; a fixed-seed chi-square test of about 2^20
draws checks the distribution against the exact float64 probabilities.  Harness streams: top_k = 1 reproduces greedy decoding bit
for bit, a seed reproduces its stream across models and resets, every fused token is the restatement's token on the fused path's
own logits, and teacher-forced fused and fused=False paths agree up to their logits' difference."""
import math

import pytest
import torch

import sample_ref as S
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
V = 128256
SEED = 0xDEADBEEF_0BADF00D


def sample(x, n, T, k, p, seed, ctr, rows=None):
    rows = x.shape[0] if rows is None else rows
    c = torch.tensor([ctr], dtype=torch.int64, device=DEV) if not torch.is_tensor(ctr) else ctr
    out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
    check(load().hqq_b200_glue_sample(ptr(x), n, x.stride(0), rows, T, k, p, seed, ptr(c), ptr(out), DTYPE_CODE[x.dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("rows", [1, 32])
def test_sample_full_vocab_matches_float64(dtype, rows):
    gen = torch.Generator(device=DEV).manual_seed(rows + DTYPE_CODE[dtype])
    x = (torch.randn(rows, V + 64, generator=gen, device=DEV) * 2.5).to(dtype)
    stats = {"rows": 0, "differ": 0}
    for i, (T, k, p) in enumerate(((0.25, 0, 1.0), (0.6, 5, 1.0), (1.0, 0, 0.9), (2.0, 50, 0.5), (0.7, 50, 0.95), (0.6, 1, 1e-3), (1.0, V, 0.9))):
        ctr = (0, 1, 2 ** 32 + 3)[i % 3]
        got = sample(x, V, T, k, p, SEED, ctr).cpu()
        lg = x[:, :V].cpu()
        u = harness.philox_uniforms(V, rows, SEED, ctr)
        for b, (t0, ok, why) in enumerate(S.accepted(lg, T, k, p, u)):
            assert int(got[b]) in ok, (T, k, p, b, int(got[b]), t0)
            stats["rows"] += 1
            stats["differ"] += int(got[b]) != t0
            if len(ok) > 1:
                stats[why] = stats.get(why, 0) + 1
    print(stats)


def planted_row(dtype):
    """A 128256-entry row with a head of 64 raised logits over a N(0, 1.5) body."""
    g = torch.Generator().manual_seed(2024)
    x = torch.randn(V, generator=g, dtype=torch.float64) * 1.5
    idx = torch.randperm(V, generator=g)[:64]
    x[idx] += torch.linspace(3.0, 9.0, 64, dtype=torch.float64)
    return x.to(dtype)


@pytest.mark.parametrize("T,k,p", [(0.6, 5, 1.0), (1.0, 0, 0.9), (0.7, 50, 0.95)])
def test_sample_distribution_chi_square(T, k, p):
    from scipy.stats import chisquare
    row = planted_row(torch.float16)
    R, C = 4096, 256
    x = row.to(DEV).view(1, V).expand(R, V).contiguous()
    counts = torch.zeros(V, dtype=torch.int64, device=DEV)
    c = torch.zeros(1, dtype=torch.int64, device=DEV)
    out = torch.empty(R, dtype=torch.int64, device=DEV)
    lib = load()
    for ctr in range(C):
        c.fill_(ctr)
        check(lib.hqq_b200_glue_sample(ptr(x), V, V, R, T, k, p, SEED, ptr(c), ptr(out), DTYPE_CODE[torch.float16], stream_ptr(DEV)))
        counts += torch.bincount(out, minlength=V)
    counts = counts.cpu().double()
    lv = row.double().view(1, V)
    keep = S.keep_topp(lv, S.keep_topk(lv, k), S.fp32(T), S.fp32(p))[0]
    w = torch.where(keep, torch.exp((lv[0] - lv[0].max()) / S.fp32(T)), torch.zeros(V, dtype=torch.float64))
    prob = w / w.sum()
    assert counts[~keep].sum() == 0, "a draw outside the kept set"
    exp = prob * (R * C)
    big = exp >= 5
    obs = torch.cat([counts[big], counts[~big].sum().view(1)])
    ex = torch.cat([exp[big], exp[~big].sum().view(1)])
    if ex[-1] == 0:
        obs, ex = obs[:-1], ex[:-1]
    stat, pval = chisquare(obs.numpy(), ex.numpy())
    print(f"T {T} top_k {k} top_p {p}: kept {int(keep.sum())}, cells {len(ex)}, chi2 {stat:.1f}, p {pval:.3g}")
    assert pval >= 1e-6


def test_sample_deterministic_and_counter_moves():
    x = planted_row(torch.bfloat16).to(DEV).view(1, V).expand(8, V).contiguous()
    a = sample(x, V, 1.0, 0, 0.9, SEED, 17)
    assert torch.equal(a, sample(x, V, 1.0, 0, 0.9, SEED, 17))
    draws = {tuple(sample(x, V, 1.0, 0, 0.9, SEED, c).tolist()) for c in range(8)}
    assert len(draws) > 1


# ------------------------------------------------------------------------------------------------ harness
SHAPE = harness.LlamaShape(n_layers=2)  # Llama-3-8B-shaped, 2 layers


def model(fused, dtype, batch=1, kv_bits=16, **kw):
    return harness.DecodeModel(SHAPE, dtype=dtype, device=DEV, cache_len=1024, fused=fused, seed=5, batch=batch, kv_bits=kv_bits, **kw)


def run(m, steps=12, prompt=None):
    """Prefill, then `steps` captured steps fed back: the token stream (per-step lists) and, for fused models, the (counter, logits)
    each token was drawn from."""
    if m.graph is None:
        m.capture()
    m.reset_state()
    toks, seen = [m.prefill(prompt, chunk=64).tolist()], [(0, m.last_logits.clone())]
    for _ in range(steps):
        ctr = int(m._sample_ctr.item())
        m.decode()
        torch.cuda.synchronize(DEV)
        toks.append(m.next_tok.tolist())
        if m.fused:
            seen.append((ctr, m._bufs["logits"].clone()))
    return toks, seen


def run_ref(m, prompt, forced):
    """fused=False, eagerly, fed the tokens `forced` (teacher forcing): its picks and the (counter, logits) of each."""
    m.reset_state()
    toks, seen = [m.prefill(prompt, chunk=64).tolist()], [(0, m.last_logits.clone())]
    captured = {}
    orig = harness.sample_tokens

    def spy(logits, *a, **k):
        captured["l"] = logits.clone()
        return orig(logits, *a, **k)
    harness.sample_tokens = spy
    try:
        for i in range(len(forced) - 1):
            m.tok.copy_(torch.tensor(forced[i], device=DEV))
            ctr = int(m._sample_ctr.item())
            with torch.no_grad():
                m.step()
            toks.append(m.next_tok.tolist())
            seen.append((ctr, captured["l"]))
    finally:
        harness.sample_tokens = orig
    return toks, seen


CONFIGS = [(5, 1, 16), (True, 1, 16), (True, 4, 16), (5, 1, 8)]
KW = dict(do_sample=True, temperature=0.7, top_k=50, top_p=0.95, sample_seed=11)


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("fused,batch,kv_bits", CONFIGS, ids=["fused5", "fused", "batch4", "kv8"])
def test_harness_sampling(dtype, fused, batch, kv_bits):
    prompt = torch.randint(0, V, (batch, 40), generator=torch.Generator(device=DEV).manual_seed(batch), device=DEV)
    greedy, gseen = run(model(fused, dtype, batch, kv_bits), prompt=prompt)
    top1, _ = run(model(fused, dtype, batch, kv_bits, do_sample=True, top_k=1), prompt=prompt)
    # top_k = 1 is the argmax where the maximum is unique; a tied maximum (common in bf16 over 128256 logits) keeps every tied
    # element in the race, and the streams part there
    for i, (x, y) in enumerate(zip(top1, greedy)):
        if x != y:
            lg = gseen[i][1].float()
            for b in range(batch):
                if x[b] != y[b]:
                    mx = lg[b].max()
                    assert lg[b, x[b]] == mx and lg[b, y[b]] == mx, (i, b, x[b], y[b])
            break
    m = model(fused, dtype, batch, kv_bits, **KW)
    a, seen = run(m, prompt=prompt)
    assert run(model(fused, dtype, batch, kv_bits, **KW), prompt=prompt)[0] == a
    m.capture()  # re-capture, then a reset run reproduces the stream
    assert run(m, prompt=prompt)[0] == a
    assert run(model(fused, dtype, batch, kv_bits, **dict(KW, sample_seed=12)), prompt=prompt)[0] != a
    # every fused token is the restatement's token on the fused path's own logits, at the model's counter, for its row b
    for (ctr, lg), t in zip(seen, a):
        u = harness.philox_uniforms(V, batch, KW["sample_seed"], ctr)
        for b, (t0, ok, why) in enumerate(S.accepted(lg.cpu(), KW["temperature"], KW["top_k"], KW["top_p"], u)):
            assert t[b] in ok, (ctr, b, t[b], t0)
    # teacher forcing: the framework-op path picks the same token, except where its logits and the fused ones differ enough
    ref, ref_seen = run_ref(model(False, dtype, batch, kv_bits, **KW), prompt, a)
    mism = 0
    for i, (x, y) in enumerate(zip(a, ref)):
        for b in range(batch):
            if x[b] != y[b]:
                mism += 1
                assert explained(ref_seen[i], seen[i][1], x[b], y[b], b), (i, b, x[b], y[b])
    print(f"{dtype} fused={fused} batch={batch} kv_bits={kv_bits}: {mism} of {len(a) * batch} picks differ")
    assert mism <= len(a) * batch // 4, (mism, a, ref)


def explained(ref_step, fused_logits, x, y, b):
    """A differing pick x (fused) / y (framework) is allowed where the two paths' logits differ by enough to reorder the two race
    keys, or to move one of them across the top-k pivot or the top-p threshold."""
    ctr, lr = ref_step
    lr, lf = lr[b:b + 1].double().cpu(), fused_logits[b:b + 1].double().cpu()
    dl = float((lr - lf).abs().max())
    T = S.fp32(KW["temperature"])
    u = harness.philox_uniforms(V, b + 1, KW["sample_seed"], ctr)[b]
    key = lr[0] / T - torch.log(-torch.log(u))
    if abs(float(key[x] - key[y])) <= 2 * dl / T + 1e-3:
        return True
    keep_k = S.keep_topk(lr, KW["top_k"])
    edges = [float(lr[keep_k].min()), float(lr[S.keep_topp(lr, keep_k, T, S.fp32(KW["top_p"]))].min())]
    return any(abs(float(lr[0, t]) - e) <= 2 * dl for t in (x, y) for e in edges)


def test_sampling_arguments():
    for kw in ({"temperature": 0}, {"temperature": -1.0}, {"temperature": float("inf")}, {"temperature": float("nan")}, {"top_k": -1},
               {"top_k": 2.5}, {"top_p": 0}, {"top_p": 1.5}, {"sample_seed": -1}, {"sample_seed": 2 ** 64}):
        with pytest.raises(ValueError):
            harness.DecodeModel(harness.TINY, dtype=torch.float16, device=DEV, cache_len=64, n_layers=1, **kw)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp_sampling_two_gpus():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", os.path.join(root, "tools", "tp_sample_check.py")],
                       capture_output=True, text=True, cwd=root, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
