"""Per-slot sampling and penalties on the H100: hqq_b200_glue_penalize and hqq_b200_glue_sample_slots at the full vocabulary, and
DecodeModel(slot_sampling=True).

Kernels: the penalised rows are tests/penalty_ref.py's bits and the counts its counts; the per-slot sampler draws the scalar
sampler's tokens.  Harness: with every slot on the constructor's settings and neutral penalties a slot_sampling model emits the
plain do_sample model's tokens (all slots at temperature 0: the greedy model's), a mixed batch emits each uniform model's tokens
for its slots, and every token of a captured step with penalties is the restatement's token on the step's own raw logits and
token tables -- through set_sampling between replays, a fork, a release and a refill."""
import gc

import pytest
import torch

import penalty_ref
import sample_ref as S
from hqq_b200 import harness
from hqq_b200._lib import DTYPE_CODE, check, load, ptr, stream_ptr

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda", 0)
V8B = harness.LLAMA3_8B.vocab
SEED = 0x51_07_5A_3B
TINY = harness.TINY
L2 = harness.LlamaShape(n_layers=2)  # Llama-3-8B-shaped, 2 layers
# a small model the fused steps run: head_dim 128, which the decode attention and kv_bits 8 need (TINY's is 64)
SMALL = harness.LlamaShape(hidden=1024, inter=2048, n_layers=2, n_heads=8, n_kv_heads=2, vocab=2048)
SAMPLE = dict(temperature=0.7, top_k=50, top_p=0.95, sample_seed=11)


def bits(t):
    return t.contiguous().view(torch.int16)


# ------------------------------------------------------------------------------------------------ kernels
def penalize(x, T, rep, freq, pres, counts, prompt, tok):
    rows, n = x.shape[0], V8B
    out = torch.full((rows, n), float("nan"), dtype=x.dtype, device=DEV)
    check(load().hqq_b200_glue_penalize(ptr(x), n, x.stride(0), rows, T, ptr(rep), ptr(freq), ptr(pres), ptr(counts), ptr(prompt), ptr(tok), ptr(out),
                                        n, DTYPE_CODE[x.dtype], stream_ptr(DEV)))
    torch.cuda.synchronize(DEV)
    return out


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16], ids=["f16", "bf16"])
@pytest.mark.parametrize("rows,T", [(1, 1), (32, 1), (32, 4)])
def test_penalize_full_vocab_bit_exact(dtype, rows, T):
    g = torch.Generator().manual_seed(rows * 10 + T)
    slots = rows // T
    x = (torch.randn(rows, V8B + 3, generator=g, dtype=torch.float64) * 3).to(dtype)
    x[:, :64] = torch.tensor([0.0, -0.0, float("inf"), float("-inf")] * 16, dtype=dtype)
    u = torch.rand(slots, V8B, generator=g)
    counts = torch.where(u < 0.7, 0, torch.where(u < 0.85, 1, torch.randint(2, 100, (slots, V8B), generator=g))).to(torch.int32)
    prompt = (torch.rand(slots, V8B, generator=g) < 0.2).to(torch.uint8)
    rep = 0.5 + torch.rand(slots, generator=g) * 1.5
    freq = torch.randn(slots, generator=g) * 0.5
    pres = torch.randn(slots, generator=g) * 0.5
    rep[0], freq[0], pres[0] = 1.0, 0.0, 0.0  # slot 0 neutral
    tok = torch.randint(0, V8B, (slots,), generator=g)
    ref, rc = penalty_ref.penalize(x[:, :V8B], T, rep, freq, pres, counts, prompt, tok)
    cd = counts.to(DEV)
    xd = x.to(DEV)
    got = penalize(xd, T, rep.to(DEV), freq.to(DEV), pres.to(DEV), cd, prompt.to(DEV), tok.to(DEV))
    assert torch.equal(bits(got.cpu()), bits(ref))
    assert torch.equal(cd.cpu(), rc)
    assert torch.equal(bits(got[:T].cpu()), bits(x[:T, :V8B]))  # neutral: the input bits
    assert torch.equal(bits(xd.cpu()), bits(x))  # the raw rows stay untouched


def test_sample_slots_full_vocab_is_the_shared_sampler():
    """32 rows on four parameter sets (one of them greedy), step and position keys: the scalar sampler's tokens row by row, the
    argmax where the temperature is 0."""
    g = torch.Generator(device=DEV).manual_seed(5)
    rows = 32
    x = (torch.randn(rows, V8B, generator=g, device=DEV) * 2.5).half()
    sets = [(0.0, 0, 1.0), (0.6, 5, 1.0), (1.0, 0, 0.9), (0.7, 50, 0.95)]
    temp = torch.tensor([sets[r % 4][0] for r in range(rows)], dtype=torch.float32, device=DEV)
    topk = torch.tensor([sets[r % 4][1] for r in range(rows)], dtype=torch.int32, device=DEV)
    topp = torch.tensor([sets[r % 4][2] for r in range(rows)], dtype=torch.float32, device=DEV)
    ctr = torch.tensor([41], dtype=torch.int64, device=DEV)
    pos = torch.arange(rows, dtype=torch.int64, device=DEV) * 3
    seq = torch.arange(rows, dtype=torch.int64, device=DEV) + 1
    lib, st, code = load(), stream_ptr(DEV), DTYPE_CODE[torch.float16]
    for keyed in (False, True):
        out = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
        check(lib.hqq_b200_glue_sample_slots(ptr(x), V8B, V8B, rows, 1, ptr(temp), ptr(topk), ptr(topp), SEED, ptr(ctr), ptr(pos) if keyed else None,
                                             ptr(seq) if keyed else None, ptr(out), code, st))
        for i, (t, k, p) in enumerate(sets):
            want = torch.full((rows,), -1, dtype=torch.int64, device=DEV)
            if t == 0:
                want = torch.argmax(x, dim=-1)
            elif keyed:
                check(lib.hqq_b200_glue_sample_pos(ptr(x), V8B, V8B, rows, t, k, p, SEED, 1, ptr(pos), ptr(seq), ptr(want), code, st))
            else:
                check(lib.hqq_b200_glue_sample(ptr(x), V8B, V8B, rows, t, k, p, SEED, ptr(ctr), ptr(want), code, st))
            torch.cuda.synchronize(DEV)
            assert torch.equal(out[i::4], want[i::4]), (keyed, i)


# ------------------------------------------------------------------------------------------------ harness
def build(shape, fused, batch, dtype, ragged=False, **kw):
    return harness.DecodeModel(shape, dtype=dtype, device=DEV, cache_len=256, fused=fused, seed=5, batch=batch, ragged=ragged, **kw)


def prompts(shape, batch, ragged):
    g = torch.Generator(device=DEV).manual_seed(3)
    if not ragged:
        return torch.randint(0, shape.vocab, (batch, 24), generator=g, device=DEV)
    return [torch.randint(0, shape.vocab, (12 + 3 * b,), generator=g, device=DEV) for b in range(batch)]


def stream(m, prompt, steps=10):
    """Capture (once), reset, prefill, `steps` replays fed back: the token lists and the prefill's last_logits."""
    if m.graph is None:
        m.capture()
    m.reset_state()
    toks = [m.prefill(prompt, chunk=64).tolist()]
    last = m.last_logits.clone()
    for _ in range(steps):
        m.decode()
        toks.append(m.next_tok.tolist())
    torch.cuda.synchronize(DEV)
    return toks, last


F16, BF16 = torch.float16, torch.bfloat16
IDENTITY = [(SMALL, 5, 1, False, d, k) for d in (F16, BF16) for k in ("step", "position")] + \
           [(SMALL, True, 8, True, d, k) for d in (F16, BF16) for k in ("step", "position")] + \
           [(L2, 5, 1, False, F16, "step"), (L2, 5, 1, False, BF16, "position"), (L2, True, 8, True, F16, "position"), (L2, True, 8, True, BF16, "step")]


@pytest.mark.parametrize("shape,fused,batch,ragged,dtype,keys", IDENTITY,
                         ids=[f"{'small' if c[0] is SMALL else 'l2'}-{'fused5' if c[1] == 5 else 'ragged8'}-{'f16' if c[4] is F16 else 'bf16'}-{c[5]}"
                              for c in IDENTITY])
def test_slot_sampling_reproduces_the_uniform_models(shape, fused, batch, ragged, dtype, keys):
    p = prompts(shape, batch, ragged)
    kw = dict(sample_keys=keys, **SAMPLE)
    plain, plain_last = stream(build(shape, fused, batch, dtype, ragged, do_sample=True, **kw), p)
    m = build(shape, fused, batch, dtype, ragged, do_sample=True, slot_sampling=True, **kw)
    got, last = stream(m, p)
    assert got == plain
    assert torch.equal(bits(last), bits(plain_last))  # last_logits stays the raw logits
    greedy, _ = stream(build(shape, fused, batch, dtype, ragged), p)
    graph = m.graph
    for b in range(batch):
        m.set_sampling(b, temperature=0)
    assert stream(m, p)[0] == greedy
    if batch > 1:  # slots 0 .. 3 greedy, 4 .. 7 sampled: each slot emits its uniform model's tokens
        for b in range(4, batch):
            m.set_sampling(b, temperature=SAMPLE["temperature"])
        mixed = stream(m, p)[0]
        assert [t[:4] for t in mixed] == [t[:4] for t in greedy]
        assert [t[4:] for t in mixed] == [t[4:] for t in plain]
    assert m.graph is graph  # set_sampling never re-captures
    if batch == 1:  # a greedy do_sample=False slot model too
        assert stream(build(shape, fused, batch, dtype, ragged, slot_sampling=True), p)[0] == greedy
    del m
    gc.collect()
    torch.cuda.empty_cache()


class Mirror:
    """Host copies of the token tables and the checks of one captured step against the restatement."""

    def __init__(self, m):
        self.m, self.B, self.V = m, m.batch, m.shape.vocab
        self.counts = torch.zeros(self.B, self.V, dtype=torch.int32)
        self.prompt = torch.zeros(self.B, self.V, dtype=torch.uint8)
        self.exact = self.rows = 0

    def prefill(self, toks, starts):
        for b, t in enumerate(toks):
            if t is None:
                continue
            if starts[b] == 0:
                self.counts[b] = 0
                self.prompt[b] = 0
            self.prompt[b, t.cpu()] = 1

    def tokens(self, pen, got, ctr, pos, seq, rows):
        m = self.m
        temp, topk, topp = m.slot_temperature.cpu(), m.slot_top_k.cpu(), m.slot_top_p.cpu()
        c = harness.position_counter(pos.cpu(), seq.cpu()) if m.position_keys else int(ctr)
        u = harness.philox_uniforms(self.V, self.B, m.sample_seed, c)
        for b in rows:
            if float(temp[b]) == 0:
                assert int(got[b]) == int(torch.argmax(pen[b])), b
                continue
            t0, ok, _ = S.accepted(pen[b:b + 1], float(temp[b]), int(topk[b]), float(topp[b]), u[b:b + 1])[0]
            assert int(got[b]) in ok, (b, int(got[b]), t0)
            self.exact += int(got[b]) == t0
            self.rows += 1

    def penalties(self):
        m = self.m
        return m.slot_repetition.cpu(), m.slot_frequency.cpu(), m.slot_presence.cpu()

    def prefill_head(self, rows, key_pos, ctr):
        """The prefill head of `rows` (ragged: last_logits holds them in slot order): nothing counted, the prompt in the tables."""
        m = self.m
        lg = torch.zeros(self.B, self.V, dtype=m.dtype)
        lg[rows] = m.last_logits.cpu()
        pen, _ = penalty_ref.penalize(lg, 1, *self.penalties(), self.counts, self.prompt, None)
        assert torch.equal(m.counts.cpu(), self.counts) and torch.equal(m.prompt_seen.cpu(), self.prompt)
        self.tokens(pen, m.tok.cpu(), ctr, torch.tensor(key_pos), m.seq.cpu() if m.seq is not None else None, rows)

    def step(self):
        m = self.m
        tok, pos, ctr = m.tok.clone(), m.pos.clone(), m._sample_ctr.clone()
        seq = m.seq.clone() if m.seq is not None else None
        m.decode()
        torch.cuda.synchronize(DEV)
        raw = m._bufs["logits"].cpu()
        pen, counts = penalty_ref.penalize(raw, 1, *self.penalties(), self.counts, self.prompt, tok.cpu())
        assert torch.equal(m.counts.cpu(), counts)
        assert torch.equal(bits(m._bufs["pen_rows"][:, :self.V].cpu()), bits(pen))
        self.tokens(pen, m.next_tok.cpu(), ctr, pos, seq, range(self.B))
        self.counts = counts


@pytest.mark.parametrize("keys", ["step", "position"])
def test_penalties_in_the_captured_step(keys):
    """kv_bits 8, paged, ragged batch 4 on the 8-launch path, mixed settings and penalties: every replay's counts and penalised rows are
    the restatement's bits and its tokens the restatement's, through set_sampling between replays, fork, release and a refill."""
    B = 4
    m = build(SMALL, True, B, F16, ragged=True, kv_bits=8, kv_pages=32, slot_sampling=True, do_sample=True, sample_keys=keys, **SAMPLE)
    m.capture()
    graph = m.graph
    m.reset_state()
    m.set_sampling(0, temperature=0, repetition_penalty=1.3, frequency_penalty=0.2, presence_penalty=0.1)
    m.set_sampling(1, temperature=0.7, top_k=0, top_p=0.9, repetition_penalty=1.1, frequency_penalty=0.5)
    m.set_sampling(2, temperature=1.0, top_k=20, top_p=1.0, presence_penalty=0.8)
    mir = Mirror(m)
    g = torch.Generator(device=DEV).manual_seed(9)
    toks = [torch.randint(0, 64, (20 + 7 * b,), generator=g, device=DEV) for b in range(B)]  # few distinct tokens: repeats
    mir.prefill(toks, [0] * B)
    ctr = m._sample_ctr.clone()
    m.prefill(toks)
    mir.prefill_head(list(range(B)), [len(t) - 1 for t in toks], ctr)
    consumed = [[] for _ in range(B)]
    for _ in range(6):
        for b in range(B):
            consumed[b].append(int(m.tok[b]))
        mir.step()
    m.set_sampling(1, temperature=0, repetition_penalty=2.0)  # takes effect at the next replay
    m.set_sampling(3, frequency_penalty=1.5, presence_penalty=0.5)
    for _ in range(3):
        mir.step()
    assert m.graph is graph
    m.fork(1, 2)  # the continuation carries slot 1's tables
    assert torch.equal(m.counts[2], m.counts[1]) and torch.equal(m.prompt_seen[2], m.prompt_seen[1])
    mir.counts[2], mir.prompt[2] = mir.counts[1], mir.prompt[1]
    m.release(3)  # the tables stay
    assert torch.equal(m.counts.cpu(), mir.counts)
    for _ in range(3):
        mir.step()
    new = torch.randint(0, 64, (17,), generator=g, device=DEV)
    mir.prefill([new, None, None, None], [0] * B)
    ctr = m._sample_ctr.clone()
    m.prefill([new, None, None, None])  # a refill at position 0: slot 0's tables start over
    assert int(m.counts[0].sum()) == 0
    mir.prefill_head([0], [16, 0, 0, 0], ctr)
    consumed[0] = []
    for _ in range(5):
        consumed[0].append(int(m.tok[0]))
        mir.step()
    assert torch.equal(m.counts[0].cpu(), torch.bincount(torch.tensor(consumed[0]), minlength=SMALL.vocab).to(torch.int32))
    assert m.graph is graph
    print(f"{keys}: {mir.exact} of {mir.rows} sampled rows are the float64 token")
    assert mir.rows and mir.exact >= mir.rows * 9 // 10


def test_framework_step_matches_the_fused_step():
    """fused=False (the reference, stepped eagerly) fed the fused model's tokens: the same tables after every step, and each path's picks on its own
    logits are apply_penalties + argmax; picks may part only where the two paths' logits differ across a near tie."""
    B = 4
    fm = build(SMALL, True, B, F16, ragged=True, slot_sampling=True)
    rm = build(SMALL, False, B, F16, ragged=True, slot_sampling=True)
    p = prompts(SMALL, B, True)
    fm.capture()
    for m in (fm, rm):
        m.reset_state()
        for b in range(B):
            m.set_sampling(b, repetition_penalty=1.2 + 0.1 * b, frequency_penalty=0.3, presence_penalty=0.2 * b)
    ft, rt = fm.prefill(p), rm.prefill(p)
    for m, t in ((fm, ft), (rm, rt)):
        pen = harness.apply_penalties(m.last_logits, m.counts, m.prompt_seen, m.slot_repetition, m.slot_frequency, m.slot_presence)
        assert torch.equal(t, torch.argmax(pen, dim=-1))
    rm.tok.copy_(fm.tok)
    mism = 0
    for i in range(10):
        fm.decode()
        with torch.no_grad():
            rm.step()
        torch.cuda.synchronize(DEV)
        assert torch.equal(fm.counts, rm.counts), i
        mism += int((fm.next_tok != rm.next_tok).sum())
        fm.tok.copy_(fm.next_tok)
        rm.tok.copy_(fm.next_tok)
    print(f"{mism} of {10 * B} picks differ between the fused and framework steps")
    assert mism <= 10 * B // 8


def test_set_sampling_arguments():
    m = build(TINY, 5, 1, F16, slot_sampling=True)
    bad = [dict(temperature=-1.0), dict(temperature=float("inf")), dict(temperature=float("nan")), dict(temperature="1"), dict(temperature=1e39),
           dict(top_k=-1), dict(top_k=2.5), dict(top_p=0), dict(top_p=1.5), dict(top_p=float("nan")), dict(repetition_penalty=0),
           dict(repetition_penalty=-1.0), dict(repetition_penalty=1e-46), dict(repetition_penalty=float("inf")), dict(frequency_penalty=float("nan")),
           dict(presence_penalty=float("-inf")), dict(presence_penalty=1e39)]
    before = [t.clone() for t in (m.slot_temperature, m.slot_top_k, m.slot_top_p, m.slot_repetition, m.slot_frequency, m.slot_presence)]
    for kw in bad:
        with pytest.raises(ValueError):
            m.set_sampling(0, temperature=0.5, **kw) if "temperature" not in kw else m.set_sampling(0, top_k=3, **kw)
    for b in (-1, 1, 0.0):
        with pytest.raises(ValueError):
            m.set_sampling(b, temperature=0.5)
    after = (m.slot_temperature, m.slot_top_k, m.slot_top_p, m.slot_repetition, m.slot_frequency, m.slot_presence)
    assert all(torch.equal(x, y) for x, y in zip(before, after))  # a rejected call writes nothing
    m.set_sampling(0, temperature=0, top_k=7, top_p=0.5, repetition_penalty=1.5, frequency_penalty=-0.5, presence_penalty=2)
    assert [float(m.slot_temperature[0]), int(m.slot_top_k[0]), float(m.slot_top_p[0]), float(m.slot_repetition[0]), float(m.slot_frequency[0]),
            float(m.slot_presence[0])] == [0.0, 7, 0.5, 1.5, -0.5, 2.0]
    with pytest.raises(ValueError, match="slot_sampling"):
        build(TINY, 5, 1, F16).set_sampling(0, temperature=0.5)


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_tp_slot_sampling_two_gpus():
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-m", "torch.distributed.run", "--nproc_per_node=2", os.path.join(root, "tools", "tp_slot_sampling_check.py")],
                       capture_output=True, text=True, cwd=root, timeout=900)
    assert r.returncode == 0, r.stdout[-3000:] + r.stderr[-3000:]
