"""The fp16 attention kernels held to error bounds derived from their roundings, and to exact results where the arithmetic is exact:
hi3d_attention_d64_tc5 (every variant, MUFU and FMA-cubic exponentials), the mma.sync d64 kernel, hi3d_attention_d80_tc5,
hi3d_attention_d512_tc5 and hi3d_temporal_attention_d64.

Roundings, as the kernels' sources write them (attn_softmax.cuh, attn_tc5.cu, attn.cu, attn_d80_tc5.cu, attn512_tc5.cu):
  S      fp16 q * k products (exact in fp32) summed by the tensor cores into fp32, d / 16 k16 steps.
  c      scale * 1.4426950408889634f rounded to fp32; the reference uses this c, p_k = 2^(c (s_k - max s)).
  x      fl(fl(s c) - fl(m c)) in fp32.
  exp    ex2.approx.ftz (MUFU, tc5 d64) or exp2f (mma d64, d80, d512, temporal): about 2^-22 relative, taken as 2^-21; under
         emulation (tc5 d64, hi3d_attention_tc5_set_exp_emulation(4)) every P is exp2_fma's cubic: 1.55e-4 measured over
         [0, 1) with its fp32 Horner steps, taken as 1.6e-4.  The correction factor of the online softmax is always MUFU / exp2f.
  P      rounded to fp16 for P V: 2^-11 relative, or 2^-25 absolute below fp16's normal range.
  l      the row sum, fp32, of the UNROUNDED P: BN / 4 adds per key tile and thread, one multiply-add per tile, two shuffles.
  O      P V on the tensor cores into fp32, rescaled by the correction once per key tile, then O * (1 / l), then fp16.

Bound per output element (reference_and_bound), with p_k the exact weights, l = sum_k p_k, ref = sum_k p_k v_k / l:
  e_k  = expm1(ln2 c |dS_k| + ln2 |dx_k|) + eps_exp + eps_corr    relative error of p_k common to O and l
         |dS_k| <= 2^-23 (2 ceil(d / 16) + 1) sum_d |q_d k_d|      two roundings per k16 step of the S accumulation
         |dx_k| <= 2^-23 (|c s_k| + |c m|)                        the fp32 rounding of x and of m c
         eps_corr = (n_tiles - 1) 2^-21 + ln2 2^-23 c (m - min_k s_k)   every rescale of the earlier tiles
  err  = [ sum_k max(2^-11 p'_k, 2^-25) |v_k|                      P rounded to fp16, in O only
         + sum_k p_k e_k (|v_k| + |ref|)                           an error common to O and l moves O / l by at most this
         + g_O sum_k p'_k |v_k| (1 + 2^-10) ] / l                  P V accumulation, g_O = 2^-23 (2 ceil(L / 16) + 2 n_tiles + 2)
         + g_l |ref|                                               l accumulation and 1 / l, g_l = 2^-24 (BN / 4 + 2 n_tiles + 4)
  bound = (1 + 2^-11) err + 2^-11 |ref| + 2^-25                    fp16 output
with p'_k = p_k (1 + e_k).  Where every score is an integer and c = 1 exactly (exact P), x and S are exact and P is a power of
two: the S, x and P-rounding terms drop, leaving accumulation, exponential and output rounding.

Exact tests: one-hot keys (each row must return its target key's V row bit for bit), a key census with q = 0 (P = 1, l = L,
O a sum of powers of two: the output is fl16(fl32(O) * fl32(1 / L)) bit for bit), image and head independence, repeatability and
NaN guard rows after every output.  Each test prints its worst |err| / bound, and the module prints the table at the end."""
import math

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops  # noqa: E402

DEV = "cuda"
F16 = torch.float16
GUARD = 256
LN2 = math.log(2.0)
U = 2.0 ** -24
EXP_MUFU = 2.0 ** -21
EXP_FMA = 1.6e-4
TC5_BN = (64, 64, 64, 128, 128, 64, 128)          # attn_tc5.cu FA_VARIANT_BN
TC5_DEFAULT = (6, 0)                               # FA_VARIANT_DEFAULT, FA_EMU_DEFAULT
RATIOS = {}


# ---- kernels and layouts -------------------------------------------------------------------------------------------------------
class Kernel:
    """One attention entry point: head dim d, key tile bn (the online softmax's tile), P's exponential error."""

    def __init__(self, name, d, bn, exp_err, fn):
        self.name, self.d, self.bn, self.exp_err, self.fn = name, d, bn, exp_err, fn

    def __repr__(self):
        return self.name


def _tc5(variant, emu):
    def run(qkv, lay, out, scale):
        lib = _native.load()
        _native.check(lib.hi3d_attention_tc5_set_variant(variant), "set_variant")
        _native.check(lib.hi3d_attention_tc5_set_exp_emulation(emu), "set_exp_emulation")
        try:
            ops.attention_d64(qkv, lay.n_img, lay.L, lay.heads, out, scale, engine="tc5")
        finally:
            _native.check(lib.hi3d_attention_tc5_set_variant(TC5_DEFAULT[0]), "set_variant")
            _native.check(lib.hi3d_attention_tc5_set_exp_emulation(TC5_DEFAULT[1]), "set_exp_emulation")
    return Kernel(f"d64 tc5 v{variant} emu{emu}", 64, TC5_BN[variant], EXP_FMA if emu else EXP_MUFU, run)


TC5_ALL = [_tc5(v, e) for v in range(7) for e in (0, 4)]
TC5_DEF = [k for k in TC5_ALL if k.name == "d64 tc5 v6 emu0"][0]
MMA = Kernel("d64 mma", 64, 64, EXP_MUFU,
             lambda qkv, lay, out, scale: ops.attention_d64(qkv, lay.n_img, lay.L, lay.heads, out, scale, engine="mma"))
D64_ALL = TC5_ALL + [MMA]
D80 = Kernel("d80 tc5", 80, 64, EXP_MUFU, lambda qkv, lay, out, scale: ops.attention_d80(qkv, lay.n_img, lay.L, lay.heads, out, scale))
D512 = Kernel("d512 tc5", 512, 64, EXP_MUFU, lambda qkv, lay, out, scale: ops.attention_d512(qkv, lay.n_img, lay.L, out, scale))
TEMPORAL = Kernel("temporal", 64, 16, EXP_MUFU,
                  lambda qkv, lay, out, scale: ops.temporal_attention_d64(qkv, lay.B, lay.T, lay.S, lay.heads, out, scale))


class Spatial:
    """[n_img * L, parts * heads * d] q|k|v / out matrices as G = n_img * heads groups (image-major) of n = L rows."""

    def __init__(self, n_img, L, heads, d):
        self.n_img, self.L, self.heads, self.d = n_img, L, heads, d
        self.G, self.n, self.rows, self.C = n_img * heads, L, n_img * L, heads * d

    def view(self, x, parts):               # [parts, n_img, heads, L, d], a view
        return x[:self.rows].view(self.n_img, self.L, parts, self.heads, self.d).permute(2, 0, 3, 1, 4)

    def split(self, x, parts):              # [parts, G, n, d]
        return self.view(x, parts).reshape(parts, self.G, self.n, self.d)

    def put(self, x, part, t):              # write group tensor t [G, n, d] into part `part` of x
        self.view(x, 3)[part] = t.view(self.n_img, self.heads, self.L, self.d)

    def join(self, *ts):
        x = torch.stack(ts).view(len(ts), self.n_img, self.heads, self.L, self.d).permute(1, 3, 0, 2, 4)
        return x.reshape(self.rows, len(ts) * self.C).contiguous()


class Temporal:
    """Rows (clip b, frame t, pixel s) as G = B * S * heads groups of n = T frames."""

    def __init__(self, B, T, S, heads):
        self.B, self.T, self.S, self.heads, self.d = B, T, S, heads, 64
        self.G, self.n, self.rows, self.C = B * S * heads, T, B * T * S, heads * 64

    def view(self, x, parts):               # [parts, B, S, heads, T, 64]
        return x[:self.rows].view(self.B, self.T, self.S, parts, self.heads, 64).permute(3, 0, 2, 4, 1, 5)

    def split(self, x, parts):
        return self.view(x, parts).reshape(parts, self.G, self.n, 64)

    def put(self, x, part, t):
        self.view(x, 3)[part] = t.view(self.B, self.S, self.heads, self.T, 64)

    def join(self, *ts):
        x = torch.stack(ts).view(len(ts), self.B, self.S, self.heads, self.T, 64).permute(1, 4, 2, 0, 3, 5)
        return x.reshape(self.rows, len(ts) * self.C).contiguous()


def launch(kern, lay, qkv, scale):
    """The kernel into a NaN-filled buffer with GUARD rows past the output, which must stay NaN; returns the output rows."""
    buf = torch.full((lay.rows + GUARD, lay.C), float("nan"), dtype=F16, device=DEV)
    kern.fn(qkv, lay, buf[:lay.rows], scale)
    assert bool(buf[lay.rows:].isnan().all()), f"{kern.name}: stores past the last output row"
    return buf[:lay.rows]


# ---- reference and bound -------------------------------------------------------------------------------------------------------
def c_log2(scale):
    """The kernels' scale_log2 = scale * 1.4426950408889634f, in fp32."""
    return float(np.float32(np.float32(scale) * np.float32(1.4426950408889634)))


def reference_and_bound(q, k, v, scale, kern, exact=False):
    """q [g, m, d] (the query rows checked), k [g, n, d], v [g, n, dv] -> float64 ref and bound [g, m, dv] (module docstring)."""
    q, k, v = q.double(), k.double(), v.double()
    n, d = k.shape[1], k.shape[2]
    c = c_log2(scale)
    nt = -(-n // kern.bn)
    s = q @ k.transpose(1, 2)
    m = s.amax(2, keepdim=True)
    p = torch.exp2(c * (s - m))
    l = p.sum(2, keepdim=True)
    av = v.abs()
    ref = (p @ v) / l
    e = kern.exp_err + (nt - 1) * EXP_MUFU + LN2 * 2 * U * c * (m - s.amin(2, keepdim=True))
    if not exact:
        ds = 2 * U * (2 * -(-d // 16) + 1) * (q.abs() @ k.abs().transpose(1, 2))
        dx = 2 * U * c * (s.abs() + m.abs())
        e = e + torch.expm1(LN2 * (c * ds + dx))
    else:
        e = e.expand_as(p)
    pe = p * e
    p1 = p + pe
    g_o = 2 * U * (2 * -(-n // 16) + 2 * nt + 2)
    g_l = U * (kern.bn // 4 + 2 * nt + 4)
    err = pe @ av + pe.sum(2, keepdim=True) * ref.abs() + g_o * (1 + 2.0 ** -10) * (p1 @ av)
    if not exact:
        err += torch.clamp_min(2.0 ** -11 * p1, 2.0 ** -25) @ av
    err = err / l + g_l * ref.abs()
    return ref, (1 + 2.0 ** -11) * err + 2.0 ** -11 * ref.abs() + 2.0 ** -25


def check_bound(kern, test, out_g, q, k, v, scale, rows=None, exact=False):
    """out_g [G, n, dv] of the kernel against reference_and_bound on query rows `rows` (default all), in chunks; returns and
    records the worst |err| / bound."""
    G, n = k.shape[:2]
    rows = torch.arange(q.shape[1], device=DEV) if rows is None else rows.to(DEV)
    m = len(rows)
    budget = 1 << 22
    gc = max(1, budget // (m * n))
    rc = m if m * n <= budget else max(1, budget // n)
    worst = 0.0
    for g0 in range(0, G, gc):
        for r0 in range(0, m, rc):
            rr = rows[r0:r0 + rc]
            ref, bound = reference_and_bound(q[g0:g0 + gc, rr], k[g0:g0 + gc], v[g0:g0 + gc], scale, kern, exact)
            d = (out_g[g0:g0 + gc, rr].double() - ref).abs()
            bad = ~(d <= bound)                                  # NaN fails too
            assert not bool(bad.any()), (f"{kern.name} {test}: {int(bad.sum())} of {bad.numel()} outside the bound (groups "
                                         f"{g0}..); worst excess {float((d - bound).nan_to_num(float('inf')).max()):.3e}, "
                                         f"max |err| {float(d.max()):.3e}")
            worst = max(worst, float((d / bound).max()))
    key = (kern.name, test)
    RATIOS[key] = max(RATIOS.get(key, 0.0), worst)
    print(f"[attention bounds] {kern.name:18s} {test:28s} worst |err| / bound {worst:.4f}")
    return worst


def assert_bits(kern, test, got, want):
    """got == want bit for bit ([G, n, dv] each); names the first wrong (group, row)s."""
    a, b = got.contiguous().view(torch.int16), want.contiguous().view(torch.int16)
    bad = (a != b).any(-1)
    assert not bool(bad.any()), (f"{kern.name} {test}: {int(bad.sum())} rows differ, first (group, row) "
                                 f"{bad.nonzero()[:6].tolist()}")
    RATIOS.setdefault((kern.name, test), 0.0)


@pytest.fixture(scope="module", autouse=True)
def _report():
    yield
    if RATIOS:
        print("\n[attention bounds] worst |err| / bound per kernel and test (0 = exact, checked bit for bit)")
        for (name, test), r in sorted(RATIOS.items()):
            print(f"  {name:18s} {test:28s} {r:.4f}")


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _randn(shape, g, std=1.0, mean=0.0):
    return (torch.randn(shape, generator=g, device=DEV) * std + mean).to(F16)


# ---- 2. key-by-key wiring (exact) ----------------------------------------------------------------------------------------------
def _f16_table():
    """Every normal fp16 value, both signs, in a fixed shuffled order: distinct, finite, and large enough that the ~2^-104
    weights of the other keys vanish next to them in fp32."""
    bits = torch.arange(0x0400, 0x7C00, dtype=torch.int32)
    bits = torch.cat([bits, bits - 0x8000])                          # - 0x8000: the negative values' int16 patterns
    bits = bits[torch.randperm(len(bits), generator=torch.Generator().manual_seed(0))]
    return bits.to(torch.int16).view(F16)


F16_TABLE = _f16_table()                                             # on the CPU: importing this module touches no GPU
PAIRS64 = torch.combinations(torch.arange(64), 2)                    # 2016 codes of two channels
PAIRS80 = torch.cartesian_prod(torch.arange(64), torch.arange(64, 80))   # one channel per S piece of d80: 1024 codes
PAIRS512 = torch.combinations(torch.arange(512), 2)


def one_hot(lay, pool, g):
    """q|k|v where row r of each group holds 24 at the two channels of its target key tgt[r] and key j at its own code's
    channels: the target scores 1152, any other key at most 576.  tgt is a random permutation (every key is one row's
    target), codes are distinct within a group, V holds distinct fp16 values per (key, column) across at least 120 keys."""
    G, n, d = lay.G, lay.n, lay.d
    codes = pool.to(DEV)[torch.rand(G, len(pool), generator=g, device=DEV).argsort(1)[:, :n]]          # [G, n, 2]
    tgt = torch.rand(G, n, generator=g, device=DEV).argsort(1)
    q = torch.zeros(G, n, d, device=DEV)
    k = torch.zeros(G, n, d, device=DEV)
    q.scatter_(2, codes.gather(1, tgt[..., None].expand(G, n, 2)), 24.0)
    k.scatter_(2, codes, 24.0)
    ar, table = torch.arange, F16_TABLE.to(DEV)
    v = table[(ar(n, device=DEV)[:, None] * d + ar(d, device=DEV) + 7919 * ar(G, device=DEV)[:, None, None]) % len(table)]
    return lay.join(q.to(F16), k.to(F16), v), v.gather(1, tgt[..., None].expand(G, n, d)), codes


def _check_one_hot(kern, lay, pool, seed):
    scale = 0.125
    assert 576 * c_log2(scale) > 26          # every other weight is below 2^-26: 0 in fp16 P, and 1 + sum of them == 1 in fp32
    qkv, want, _ = one_hot(lay, pool, _gen(seed))
    out = launch(kern, lay, qkv, scale)
    assert_bits(kern, "one-hot wiring", lay.split(out, 1)[0], want)


D64_L = [1, 63, 65, 127, 129, 191, 193, 255, 449]


@pytest.mark.parametrize("kern", D64_ALL, ids=str)
def test_one_hot_d64(kern):
    """L puts the key tail in each consumer warpgroup and at several 8-column n-tiles of both key tiles; 3 images, so every
    image's tail tile reads the next image's keys (whose codes can equal a target's)."""
    for L in D64_L:
        _check_one_hot(kern, Spatial(3, L, 2, 64), PAIRS64, L)


def test_one_hot_d80():
    """Codes pair a channel of the 64-column SWIZZLE_128B piece with one of the 16-column SWIZZLE_32B piece: without the fifth
    k16 step every key sharing the first channel ties with the target.  Columns 64..79 of V are compared like the others."""
    for L in [1, 63, 64, 65, 257, 1000]:
        _check_one_hot(D80, Spatial(3, L, 2, 80), PAIRS80, L)


def test_one_hot_d512():
    """Codes of two of the 512 channels: the selecting channels fall in each of the eight 64-column chunks of S; both 256-column
    value halves are compared."""
    for L, n_img in [(128, 3), (256, 2), (4096, 2)]:
        lay = Spatial(n_img, L, 1, 512)
        qkv, want, codes = one_hot(lay, PAIRS512, _gen(L))
        assert set((codes // 64).unique().tolist()) == set(range(8))
        out = launch(D512, lay, qkv, 0.125)
        assert_bits(D512, "one-hot wiring", lay.split(out, 1)[0], want)


def test_one_hot_temporal():
    """Every T, 2 clips, a ragged pixel count, a random permutation of the frames as targets per (clip, pixel, head)."""
    for T in range(1, 17):
        _check_one_hot(TEMPORAL, Temporal(2, T, 37, 2), PAIRS64, T)


# ---- 3. key census (exact) -----------------------------------------------------------------------------------------------------
POW = (8.0, 2.0, 0.5, 0.125)          # distinct powers of two within 6 bits: any column sum of them is exact in fp32
BIG = 16384.0


def _census(kern, lay, big_last=False):
    """q = 0: every score is 0, P = 1 on both exponential pipes, l = L.  Per call, key j of group g is live when
    (j + g) % ncalls == call: it adds POW[i // dv] to column (i + 13 g) % dv, i = j // ncalls, so a column holds at most one key
    per power and its sum is exact; the calls together make every key of every group live once.  The output must be
    fl16(fl32(sum) * fl32(1 / L)) bit for bit, as the kernels finish (O * (1.f / l)).  big_last: the last image's V is BIG
    everywhere, so a key of it counted by the image before moves that image's outputs by orders of magnitude, and its own tail
    is TMA zeros, where an extra key changes l by more than an fp16 ulp."""
    G, n, dv = lay.G, lay.n, lay.d
    per = dv * len(POW)
    ncalls = -(-n // per)
    g = _gen(n)
    qkv = lay.join(torch.zeros(G, n, lay.d, dtype=F16, device=DEV), _randn((G, n, lay.d), g), torch.zeros(G, n, dv, dtype=F16, device=DEV))
    j = torch.arange(n, device=DEV)[None]
    gi = torch.arange(G, device=DEV)[:, None]
    i = (j // ncalls).expand(G, n)
    col = (i + 13 * gi) % dv
    pw = torch.tensor(POW, device=DEV)[i // dv]
    inv = torch.tensor(1.0, dtype=torch.float32) / torch.tensor(float(n), dtype=torch.float32)
    n_big = lay.heads if big_last else 0
    for call in range(ncalls):
        v = torch.zeros(G, n, dv, device=DEV)
        v.scatter_(2, col[..., None], torch.where((j + gi) % ncalls == call, pw, 0.0)[..., None])
        if n_big:
            v[G - n_big:] = BIG
        lay.put(qkv, 2, v.to(F16))
        want = (v.sum(1, keepdim=True) * inv.to(DEV)).to(F16).expand(G, n, dv)
        out = launch(kern, lay, qkv, 0.125)
        assert_bits(kern, "census", lay.split(out, 1)[0], want)


@pytest.mark.parametrize("kern", D64_ALL + [D80], ids=str)
def test_census(kern):
    """Every key of 2 images x 2 heads at L = 4096 and 16384 (multiples of every key tile), and tails on the last image."""
    for L in (4096, 16384):
        _census(kern, Spatial(2, L, 2, kern.d))
    for L in (1, 65, 100, 200):
        _census(kern, Spatial(2, L, 2, kern.d), big_last=True)


def test_census_d512():
    _census(D512, Spatial(2, 4096, 1, 512))
    _census(D512, Spatial(3, 128, 1, 512), big_last=True)


def test_census_temporal():
    for T in range(1, 17):
        _census(TEMPORAL, Temporal(2, T, 37, 2))


# ---- 4. exact P ----------------------------------------------------------------------------------------------------------------
LN2_F32 = float(np.float32(LN2))


def _exact_p(kern, lay, seed):
    """Scale = fp32(ln 2), so c = 1 exactly; q has eight ones per group row and k entries in {-1, 0, 1}: scores are integers
    in [-8, 8], within 16 of the row maximum, so every P = 2^(s - m) >= 2^-16 is a power of two, exact in fp16."""
    assert c_log2(LN2_F32) == 1.0
    G, n, d = lay.G, lay.n, lay.d
    g = _gen(seed)
    q = torch.zeros(G, n, d, device=DEV)
    q.scatter_(2, torch.rand(G, n, d, generator=g, device=DEV).argsort(2)[..., :8], 1.0)
    k = torch.randint(-1, 2, (G, n, d), generator=g, device=DEV).float()
    v = _randn((G, n, d), g)
    qkv = lay.join(q.to(F16), k.to(F16), v)
    out = launch(kern, lay, qkv, LN2_F32)
    return check_bound(kern, "exact P", lay.split(out, 1)[0], q, k, v, LN2_F32, exact=True)


@pytest.mark.parametrize("kern", D64_ALL + [D80], ids=str)
def test_exact_p(kern):
    for L in (1000, 4096):
        _exact_p(kern, Spatial(2, L, 3, kern.d), L)


def test_exact_p_d512():
    _exact_p(D512, Spatial(2, 4096, 1, 512), 4096)


def test_exact_p_temporal():
    for T in range(1, 17):
        _exact_p(TEMPORAL, Temporal(2, T, 37, 2), T)


# ---- 5. long one-sign sums -----------------------------------------------------------------------------------------------------
def _sample_rows(n, g):
    if n <= 256:
        return torch.arange(n)
    mid = torch.randperm(n - 64, generator=g)[:192] + 32
    return torch.cat([torch.arange(32), mid, torch.arange(n - 32, n)])


def _long_spatial(kern, n_img, L, heads):
    """Scores spread over a few units (q, k ~ N(0, 1), c s ~ N(0, 1.44^2)) and V = 1 + N(0, 1/16): the P V sum runs over L
    terms of one sign.  Sampled rows of the first, last and a middle (image, head)."""
    lay = Spatial(n_img, L, heads, kern.d)
    g = _gen(L + heads)
    qkv = torch.randn(lay.rows, 3 * lay.C, generator=g, device=DEV, dtype=F16)
    qkv[:, 2 * lay.C:].mul_(0.25).add_(1.0)
    out = launch(kern, lay, qkv, 0.125)
    rows = _sample_rows(L, torch.Generator().manual_seed(L))
    imgs, hs = zip(*[(0, 0), (n_img - 1, heads - 1), (n_img // 2, heads // 2)])
    imgs, hs = torch.tensor(imgs, device=DEV), torch.tensor(hs, device=DEV)
    q, k, v = lay.view(qkv, 3)[:, imgs, hs]
    return check_bound(kern, f"one-sign {n_img}x{L}x{heads}", lay.view(out, 1)[0, imgs, hs], q, k, v, 0.125, rows=rows)


UNET_SHAPES = [(32, 16384, 5), (32, 4096, 10), (32, 1024, 20), (32, 256, 20)]


@pytest.mark.parametrize("kern", [TC5_DEF, MMA], ids=str)
@pytest.mark.parametrize("n_img,L,heads", UNET_SHAPES)
def test_one_sign_unet_shapes(kern, n_img, L, heads):
    _long_spatial(kern, n_img, L, heads)


def test_one_sign_d512():
    _long_spatial(D512, 2, 16384, 1)


def test_one_sign_temporal():
    lay = Temporal(2, 16, 4096, 5)
    g = _gen(16)
    qkv = torch.randn(lay.rows, 3 * lay.C, generator=g, device=DEV, dtype=F16)
    qkv[:, 2 * lay.C:].mul_(0.25).add_(1.0)
    out = launch(TEMPORAL, lay, qkv, 0.125)
    q, k, v = lay.split(qkv, 3)
    check_bound(TEMPORAL, "one-sign 2x16x4096x5", lay.split(out, 1)[0], q, k, v, 0.125)


# ---- 6. masking, independence, guards, repeatability ---------------------------------------------------------------------------
def _masking(kern, lay, seed):
    """Random q|k|v; the queries of even images carry a 1 in the last channel and the keys of odd images 1000 there: the next
    image's keys, which an even image's tail tile reads, score about +1000 against its queries.  Masking has to happen
    before the row maximum for the output to stay within the bound."""
    G, n, d = lay.G, lay.n, lay.d
    g = _gen(seed)
    q, k, v = _randn((G, n, d), g), _randn((G, n, d), g), _randn((G, n, d), g)
    img = torch.arange(G, device=DEV) // lay.heads
    q[..., d - 1] = torch.where(img % 2 == 0, 1.0, 0.0).to(F16)[:, None]
    k[img % 2 == 1, :, d - 1] = 1000.0
    qkv = lay.join(q, k, v)
    out = launch(kern, lay, qkv, 0.125)
    return check_bound(kern, "masked next-image keys", lay.split(out, 1)[0], q, k, v, 0.125)


@pytest.mark.parametrize("kern", D64_ALL, ids=str)
def test_masking_d64(kern):
    for L in D64_L:
        _masking(kern, Spatial(3, L, 2, 64), L)


def test_masking_d80():
    for L in [1, 63, 64, 65, 257, 1000]:
        _masking(D80, Spatial(3, L, 2, 80), L)


def _independence(kern, lay, one, sub_rows, heads_of):
    """Two runs are bit-identical; each image (clip) alone equals itself inside the batch; rewriting image i + 1's q|k|v leaves
    image i bit-identical; each head alone equals its column block of the multi-head run."""
    g = _gen(lay.rows)
    qkv = _randn((lay.rows, 3 * lay.C), g)
    a = launch(kern, lay, qkv, 0.125)
    b = launch(kern, lay, qkv, 0.125)
    assert torch.equal(a.view(torch.int16), b.view(torch.int16)), f"{kern.name}: two runs differ"
    n_part = len(sub_rows)
    for i, r in enumerate(sub_rows):
        alone = launch(kern, one, qkv[r].contiguous(), 0.125)
        assert torch.equal(alone.view(torch.int16), a[r].view(torch.int16)), f"{kern.name}: part {i} alone differs"
        if i + 1 < n_part:
            other = qkv.clone()
            nxt = sub_rows[i + 1]
            other[nxt] = _randn(other[nxt].shape, g, std=3.0)
            other[nxt, lay.C:2 * lay.C] = 1000.0                      # keys that would dominate any row that counted them
            c = launch(kern, lay, other, 0.125)
            assert torch.equal(c[r].view(torch.int16), a[r].view(torch.int16)), \
                f"{kern.name}: rewriting part {i + 1} changed part {i}"
    if heads_of is not None and lay.heads > 1:
        d = lay.d
        for h in range(lay.heads):
            cols = torch.cat([torch.arange(p * lay.C + h * d, p * lay.C + (h + 1) * d) for p in range(3)]).to(DEV)
            alone = launch(kern, heads_of, qkv[:, cols].contiguous(), 0.125)
            assert torch.equal(alone.view(torch.int16), a[:, h * d:(h + 1) * d].contiguous().view(torch.int16)), \
                f"{kern.name}: head {h} alone differs from its column block"
    RATIOS.setdefault((kern.name, "independence"), 0.0)


def _spatial_independence(kern, n_img, L, heads):
    lay = Spatial(n_img, L, heads, kern.d)
    _independence(kern, lay, Spatial(1, L, heads, kern.d), [slice(i * L, (i + 1) * L) for i in range(n_img)],
                  Spatial(n_img, L, 1, kern.d))


@pytest.mark.parametrize("kern", D64_ALL, ids=str)
def test_independence_d64(kern):
    for L in (193, 449):
        _spatial_independence(kern, 3, L, 3)


def test_independence_d80_d512():
    for L in (65, 257):
        _spatial_independence(D80, 3, L, 3)
    _spatial_independence(D512, 3, 384, 1)


def test_independence_temporal():
    B, T, S, heads = 3, 7, 37, 2
    lay = Temporal(B, T, S, heads)
    _independence(TEMPORAL, lay, Temporal(1, T, S, heads), [slice(b * T * S, (b + 1) * T * S) for b in range(B)],
                  Temporal(B, T, S, 1))
