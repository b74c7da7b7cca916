"""Exact references and per-element error bounds for the fused forward (hqq_b200_linear_fwd, routes 1-3).

A test draws its own integer levels q, scale s and zero z in the compute dtype T (`draw_layer`), packs q with the oracle and
runs a kernel.  `reference` builds the exact result from the DRAWN levels (never from an unpack of the packed tensor) in float64,
and a per-element bound that follows from the kernel's arithmetic:

    |y - y*| <= 1/2 ulp_T(y*)  [+ 1/2 ulp_T for the bias's second rounding]  +  d * 2^-23 * A

  route 1 (mma.sync on exact levels planted as OFF + q in 16-bit lanes; s and z applied per group in fp32):
      y* = sum_k x_k (q_k - z_g) s_g                  A = sum_g |s_g| (OFF + 2^nbits - 1 + |z_g|) sum_{k in g} |x_k|
      d  = GS/16 + ceil(K / (8 GS)) + 12               (OFF = 1024 fp16, 128 bf16: the planted offset, so its cancellation
                                                        is inside the bound)
  routes 2 and 3 (tensor cores on W_r = T(T(q - z) * s), the reference's two roundings, quantize.py):
      y* = sum_k x_k W_r[n, k]                        A = sum_k |x_k| |W_r[n, k]|        d = K/16 + ksplit + 4

2^-23 rather than the fp32 unit roundoff 2^-24 allows for tensor-core accumulation that truncates.  `check` returns the largest
err / bound and fails past 1; `negative_controls` builds three defective outputs from the same data (a zero one level off, two
rows of different slabs swapped, the last 256-k unit dropped) that the same comparison must reject.

Everything is torch and runs on whatever device the tensors live on; float64 work is done in row chunks (`CHUNK` elements of W at
a time) so a full-size layer stays far below 1 GB on a shared card."""
import math

import torch

from oracle import hqq_oracle as O

OFF = {torch.float16: 1024.0, torch.bfloat16: 128.0}
MANT = {torch.float16: 10, torch.bfloat16: 7}
EMIN = {torch.float16: -14, torch.bfloat16: -126}
CHUNK = 1 << 24
EPS_ACC = 2.0 ** -23


def ulp(v: torch.Tensor, dtype) -> torch.Tensor:
    """Spacing of `dtype` numbers in the binade of |v| (float64; subnormal spacing below the normal range)."""
    a = v.abs().to(torch.float64)
    e = torch.floor(torch.log2(torch.clamp(a, min=2.0 ** EMIN[dtype])))
    return torch.pow(2.0, e - MANT[dtype])


def round_to(v: torch.Tensor, dtype) -> torch.Tensor:
    """float64 -> dtype with ONE round-to-nearest-even (a float64 -> float32 -> dtype cast may round twice)."""
    v = v.to(torch.float64)
    u = ulp(v, dtype)
    return (torch.round(v / u) * u).to(dtype)  # v / u is exact (u is a power of two); torch.round ties to even


class Layer:
    """Levels q (the grouped view [R, C] of the reference, unpacked), scale / zero in T ([R, 1] for axis 1, [1, C] for axis 0) and
    the packed tensor the kernels read (oracle.PACK: bit-exact with ops.pack)."""

    def __init__(self, q, s, z, N, K, gs, nbits, axis, dtype, bias=None, pack=None):
        self.q, self.s, self.z, self.N, self.K, self.gs, self.nbits, self.axis, self.dtype = q, s, z, N, K, gs, nbits, axis, dtype
        self.bias = bias
        self.G = N * K // gs
        if pack is None:
            self.W_q = torch.from_numpy(O.PACK[O.BIT_TO_PACKING[nbits]](q.cpu().numpy())).to(q.device)
        else:  # ops.pack on the GPU: bit-exact with the oracle (tests/test_bitpack_gpu.py), and quick at full size
            self.W_q = pack(q, nbits)

    @property
    def device(self):
        return self.q.device

    def meta_index(self, n0, n1):
        """Index into the flat scale / zero of every element of W rows n0..n1."""
        f = torch.arange(n0, n1, device=self.device)[:, None] * self.K + torch.arange(self.K, device=self.device)[None]
        return f // self.gs if self.axis == 1 else f % self.G

    def rows(self, n0, n1, exact, z=None):
        """W[n0:n1] in float64: (q - z) s exactly (route 1), or T(T(q - z) s) (routes 2 and 3, the reference's dequantize)."""
        z = self.z if z is None else z
        q = self.q.reshape(-1)[n0 * self.K:n1 * self.K].reshape(n1 - n0, self.K)
        idx = self.meta_index(n0, n1)
        s, zz = self.s.reshape(-1)[idx], z.reshape(-1)[idx]
        if exact:
            return (q.to(torch.float64) - zz.to(torch.float64)) * s.to(torch.float64)
        return ((q.to(self.dtype) - zz) * s).to(torch.float64)

    def route1_coef(self, n0, n1):
        """|s| (OFF + 2^nbits - 1 + |z|) per element: the magnitude the route-1 accumulators carry per unit of |x|."""
        idx = self.meta_index(n0, n1)
        s, z = self.s.reshape(-1)[idx].to(torch.float64), self.z.reshape(-1)[idx].to(torch.float64)
        return s.abs() * (OFF[self.dtype] + 2 ** self.nbits - 1 + z.abs())

    def dequantized(self):
        """T(T(q - z) s) as [N, K] in T (what layer.dequantize() must return bit for bit)."""
        return ((self.q.to(self.dtype) - self.z) * self.s).reshape(self.N, self.K)

    def chunks(self):
        step = max(1, CHUNK // self.K)
        for n0 in range(0, self.N, step):
            yield n0, min(self.N, n0 + step)


def generator(seed, device):
    return torch.Generator(device=device).manual_seed(int(seed))


def draw_layer(gen, N, K, nbits, gs, dtype, axis=1, bias=False, pack=None):
    """Random levels, scale in [2e-3, 1.2e-2), zero in [0, 2^nbits - 1) (both rounded to T), optional bias ~ N(0, 0.1^2) in T,
    on the generator's device."""
    dev = gen.device
    R, C = (N * K // gs, gs) if axis == 1 else (gs, N * K // gs)
    sh = (R, 1) if axis == 1 else (1, C)
    q = torch.randint(0, 2 ** nbits, (R, C), generator=gen, device=dev, dtype=torch.uint8)
    s = (torch.rand(sh, generator=gen, device=dev, dtype=torch.float64) * 0.01 + 2e-3).to(dtype)
    z = (torch.rand(sh, generator=gen, device=dev, dtype=torch.float64) * (2 ** nbits - 1)).to(dtype)
    b = (torch.randn(N, generator=gen, device=dev, dtype=torch.float64) * 0.1).to(dtype) if bias else None
    return Layer(q, s, z, N, K, gs, nbits, axis, dtype, b, pack)


def draw_x(gen, M, K, gs, dtype):
    """N(0, 1) activations, except that the last group of K is 'hot': same-signed and about four times larger.  The defects the
    controls model (a zero one level off in that group, the last 256-k unit dropped) then move an output by far more than the
    bound even at K = 28672, where the route-1 bound, which carries the planted offset OFF * sum |x|, is widest."""
    x = torch.randn((M, K), generator=gen, device=gen.device, dtype=torch.float64)
    x[:, K - gs:] = 4.0 * (0.5 + x[:, K - gs:].abs())
    return x.to(dtype)


def draw_x2(gen, K, gs, dtype):
    """Second prologue operand (residual delta / SiLU multiplier): N(0, 0.5^2), positive and above 0.5 in the last group, so that the
    hot group of `draw_x` stays hot through x + x2 and silu(x) * x2."""
    x2 = torch.randn((1, K), generator=gen, device=gen.device, dtype=torch.float64) * 0.5
    x2[:, K - gs:] = 0.5 + x2[:, K - gs:].abs()
    return x2.to(dtype)


class Ref:
    """y0 = exact x @ W^T (float64, no bias), E = d * 2^-23 * A (+ slack for a rounded activation), and what to compare with."""

    def __init__(self, layer, x, route, d, y0, E):
        self.layer, self.x, self.route, self.d, self.y0, self.E = layer, x, route, d, y0, E
        self.dtype = layer.dtype
        self.bias = None if layer.bias is None else layer.bias.to(torch.float64)

    @property
    def y(self):
        return self.y0 if self.bias is None else self.y0 + self.bias

    def bound(self):
        E = self.E
        if self.bias is None:
            return E + 0.5 * ulp(self.y0.abs() + E, self.dtype)
        u1 = 0.5 * ulp(self.y0.abs() + E, self.dtype)  # T(acc), then T(T(acc) + b): the reference's second rounding
        return E + u1 + 0.5 * ulp(self.y.abs() + E + u1, self.dtype)


def route_d(route, K, gs, ksplit=1):
    if route == 1:
        return gs // 16 + math.ceil(K / (8 * gs)) + 12
    return K // 16 + ksplit + 4


def reference(layer, x, route, ksplit=1, x_slack=None):
    """Exact result and bound for y = x @ W^T (+ bias) through `route`.  x_slack [M, K] (float64, optional): how far each element
    of the activation the kernel used may be from `x` (a prologue's last-ulp flips); it widens the bound by x_slack @ |W|^T."""
    exact = route == 1
    d = route_d(route, layer.K, layer.gs, ksplit)
    x64 = x.to(torch.float64)
    ax = x64.abs()
    M = x.shape[0]
    y0 = torch.empty((M, layer.N), dtype=torch.float64, device=x.device)
    A = torch.empty_like(y0)
    slack = torch.zeros_like(y0)
    for n0, n1 in layer.chunks():
        W = layer.rows(n0, n1, exact)
        y0[:, n0:n1] = x64 @ W.T
        A[:, n0:n1] = ax @ (layer.route1_coef(n0, n1) if exact else W.abs()).T
        if x_slack is not None:
            slack[:, n0:n1] = x_slack @ W.abs().T
        del W
    return Ref(layer, x, route, d, y0, d * EPS_ACC * A + slack)


def ratio(y, ref):
    """|y - y*| / bound per element (float64)."""
    return (y.to(torch.float64) - ref.y).abs() / ref.bound()


def check(y, ref, what=""):
    """Largest err / bound; fails with the worst element when it exceeds 1 (or y is not finite)."""
    assert y.shape == ref.y0.shape, (what, tuple(y.shape), tuple(ref.y0.shape))
    r = ratio(y, ref)
    assert bool(torch.isfinite(y.to(torch.float64)).all()), f"{what}: non-finite output"
    worst = float(r.max())
    if worst > 1.0:
        i = int(r.argmax())
        m, n = divmod(i, ref.y0.shape[1])
        raise AssertionError(f"{what}: |y - y*| / bound = {worst:.3g} at (m={m}, n={n}): y = {float(y.reshape(-1)[i])!r}, "
                             f"y* = {float(ref.y.reshape(-1)[i])!r}, bound = {float(ref.bound().reshape(-1)[i]):.3g}; "
                             f"{int((r > 1).sum())} of {r.numel()} elements out of bound")
    return worst


def _output(ref, y0_defect):
    """What a kernel with the defect would store: T(acc) (+ b with a second rounding)."""
    o = round_to(y0_defect, ref.dtype)
    if ref.layer.bias is not None:
        o = o + ref.layer.bias  # T + T in T: one rounding, as the kernels do
    return o


def negative_controls(ref):
    """Defective outputs built from the same data; each must be rejected by `ratio(., ref).max() > 1`.
      zero_off_by_one   in one row, the zero of the group with the largest |sum_{k in g} x_k| shifted by one level
      rows_swapped      two output rows of different slabs (one from each half of N) exchanged
      last_unit_dropped the last 256-k unit of one row left out of the sum"""
    L, x64 = ref.layer, ref.x.to(torch.float64)
    exact = ref.route == 1
    K, gs = L.K, L.gs
    out = {}
    # (a) the group: axis 1 -> the k-group with the largest |sum x| (any token), row with the largest |s|; axis 0 -> the column k
    # with the largest |x|, group (a block of gs rows) with the largest |s|
    zf = L.z.reshape(-1).clone()
    sf = L.s.reshape(-1).to(torch.float64).abs()
    if L.axis == 1:
        g = int(x64.reshape(x64.shape[0], K // gs, gs).sum(-1).abs().amax(0).argmax())
        n = int(sf.reshape(L.N, K // gs)[:, g].argmax())
        j, rows = n * (K // gs) + g, [n]
    else:
        k = int(x64.abs().amax(0).argmax())
        per = L.G // K  # W rows between two members of one axis-0 group
        blk = int(sf[torch.arange(per, device=sf.device) * K + k].argmax())
        j, rows = blk * K + k, [blk + i * per for i in range(gs)]
    zf[j] = zf[j] + 1
    z1 = zf.reshape(L.z.shape)
    y = ref.y0.clone()
    for n in rows:
        dW = L.rows(n, n + 1, exact, z=z1) - L.rows(n, n + 1, exact)
        y[:, n] += (x64 @ dW.T)[:, 0]
    out["zero_off_by_one"] = _output(ref, y)
    # (b) rows of different slabs: slab = n // (N / F), so one row from each half of N is always two slabs apart (F >= 2) or two
    # row tiles apart (F = 1); the pair with the most different values for token 0
    h = L.N // 2
    n1 = int(ref.y0[0, :h].argmax())
    n2 = h + int(ref.y0[0, h:].argmin())
    y = ref.y0.clone()
    y[:, [n1, n2]] = y[:, [n2, n1]]
    out["rows_swapped"] = _output(ref, y)
    # (c) the last 256-k unit of the row where it contributes most
    part = torch.empty_like(ref.y0)
    for n0, n1_ in L.chunks():
        part[:, n0:n1_] = x64[:, K - 256:] @ L.rows(n0, n1_, exact)[:, K - 256:].T
    n = int(part.abs().amax(0).argmax())
    y = ref.y0.clone()
    y[:, n] -= part[:, n]
    out["last_unit_dropped"] = _output(ref, y)
    return out


def assert_controls_rejected(ref, what=""):
    """Every negative control exceeds the bound somewhere; returns the smallest max(err / bound) among them."""
    least = math.inf
    for name, y in negative_controls(ref).items():
        r = float(ratio(y, ref).max())
        assert r > 1.0, f"{what}: the comparison accepts the defect '{name}' (max err / bound = {r:.3g})"
        least = min(least, r)
    return least


# ---------------------------------------------------------------------------------------------------------------- prologues
def silu_f32(v):
    v = v.to(torch.float32)
    return v / (1.0 + torch.exp(-v))


def on_grid(t, dtype, q=16.0, lim=12.0):
    """Values on multiples of 1/q, |.| <= lim: sums of two such values and their squares are exact in T and fp32 (see
    prologue_rmsnorm)."""
    return (torch.round(t.to(torch.float64) * q) / q).clamp(-lim, lim).to(dtype)


def _spread(f, lo, hi):
    """Largest |f(v) - f(mid)| over the interval's ends, for f monotone in v: how far the kernel's value can be from the reference."""
    mid = f(1.0)
    return torch.maximum((f(lo) - mid).abs(), (f(hi) - mid).abs()), mid


def prologue_rmsnorm(x, x2, w, eps, dtype):
    """x_op 1: h = T(x + x2) (x2 may be None), xn = T(T(h * rsqrt(mean(h^2) + eps)) * w), with the float64 rsqrt.  Returns
    (h, xn, slack).  The kernel's inverse norm differs from the float64 one by the fp32 sum of squares (exact when every h is a
    multiple of 1/16 and the sum stays below 2^16, else up to K/2 * 2^-24 relative), the division and + eps (2^-24 each), rsqrtf
    (2 ulp) and the fp32 product h * inv (2^-24): together below 2^-20 relative.  xn is monotone in inv, so the kernel's xn lies
    between the values at inv (1 -/+ delta); slack is the larger distance to them (zero for all but the few elements next to a
    rounding boundary)."""
    h = x if x2 is None else (x.to(torch.float32) + x2.to(torch.float32)).to(dtype)
    hf = h.to(torch.float64)
    K = h.shape[-1]
    sq = (hf * hf).sum(dim=-1, keepdim=True)
    exact_sum = bool(torch.equal(hf * 16, torch.round(hf * 16))) and float(sq.max()) * 256 < 2 ** 24
    delta = 2.0 ** -20 + (0.0 if exact_sum else K * 2.0 ** -25)
    inv = 1.0 / torch.sqrt(sq / K + eps)
    xn_at = lambda f: (round_to(hf * (inv * f), dtype).to(torch.float32) * w.to(torch.float32)).to(dtype).to(torch.float64)  # noqa: E731
    slack, xn = _spread(xn_at, 1.0 - delta, 1.0 + delta)
    return h, xn.to(dtype), slack


def prologue_silu_mul(x, x2, dtype):
    """x_op 2: xm = T(T(silu(x)) * x2), silu in float64.  The kernel's f / (1 + __expf(-f)) is within (2 + 1.173 |f|) ulp (__expf,
    CUDA's documented bound) + 2 roundings of fp32, i.e. (5 + 1.2 |f|) 2^-23 relative, of it; slack as in prologue_rmsnorm."""
    f = x.to(torch.float64)
    sl = f / (1.0 + torch.exp(-f))
    delta = (5.0 + 1.2 * f.abs()) * 2.0 ** -23
    xm_at = lambda k: (round_to(sl * (1.0 + (k - 1.0) * delta), dtype).to(torch.float32) * x2.to(torch.float32)).to(dtype).to(torch.float64)  # noqa: E731
    slack, xm = _spread(xm_at, 0.0, 2.0)
    return xm.to(dtype), slack


def silu_mul_bound(ref_g, ref_u):
    """Bound on |T(T(silu(g)) u) - silu(g*) u*| given the bounds of g and u (|silu'| <= 1.1), plus the two roundings."""
    dt = ref_g.dtype
    g, u = ref_g.y, ref_u.y
    Bg, Bu = ref_g.bound(), ref_u.bound()
    sg = g / (1.0 + torch.exp(-g))
    s_hi = sg.abs() + 1.1 * Bg
    prod = s_hi * (u.abs() + Bu)
    return 1.1 * Bg * (u.abs() + Bu) + sg.abs() * Bu + 0.5 * ulp(s_hi, dt) * (u.abs() + Bu) + 0.5 * ulp(prod, dt), sg * u
