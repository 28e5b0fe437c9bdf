"""The frame-sharded kernels on ONE GPU, against unsharded references.

Frame sharding splits each clip's T frames over `world` ranks: rank r owns frames [r Tl, (r+1) Tl).  In the peer-memory
exchange mode four pieces of CUDA serve only the sharded step:

  A. pixel-strip temporal attention (hi3d_temporal_attention_d64_sharded): reads the other ranks' q|k|v rows and stores
     their output rows straight into their buffers;
  B. the haloed temporal GroupNorm apply (hi3d_groupnorm_apply_halo / _apply_stats with neighbour pointers): writes a
     [B, Tl + 2, HW, C] buffer, copies its first / last frame into the neighbours' halo slots and zero-fills its own slot
     at a clip boundary;
  C. the (3,1,1) temporal conv over that haloed buffer (Tin = Tl + 2, t_off = 1) on both GEMM engines;
  D. the exchange kernel (hi3d_peer_exchange): a flag barrier plus the rank-order all-reduce of the GroupNorm sums.

All of them take plain device pointers, so here a "rank" is one set of buffers in this process on this device and a "world"
is a list of them.  A-C never wait on another rank: launching the ranks one after another on one stream gives the order the
exchange kernel gives in production.  D runs rank 0 only, with every flag word preset far ahead so that it never waits.
E checks that each entry point rejects geometry it cannot serve, with real buffers sized so nothing can go out of bounds.
Every check prints its max |err|.
"""
import ctypes as C

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from hi3d_official_b200 import _native, ops, pack  # noqa: E402
from test_gemm_tc5_gpu import _close_stats, _unit_sums  # noqa: E402
from test_kernels_gpu import DEV, H, close, rnd  # noqa: E402

NAN = float("nan")
GN_UNIT = 10          # UNet channels per statistics unit at model_channels = 320


def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


class _World:
    """What the sharded entry points read of a peer.SymmBuffer: `ptr_array[r]` = rank r's buffer (all on this device)."""

    def __init__(self, bufs):
        self.bufs = bufs
        self.ptr_array = (C.c_void_p * len(bufs))(*[b.data_ptr() for b in bufs])


def _nans(rows, cols):
    return torch.full((rows, cols), NAN, dtype=H, device=DEV)


def _report(name, got, ref):
    err = float((got.float() - ref.float()).abs().max()) if got.numel() else 0.0
    print(f"[shard kernels] {name}: max|err| {err:.3e}")
    return err


def _check(got, ref, name, **kw):
    """close() plus: every value finite (close() lets a NaN through) and the max |err| printed."""
    _report(name, got, ref)
    assert bool(torch.isfinite(got.float()).all()), f"{name}: non-finite values"
    close(got, ref, name=name, **kw)


def _identical(got, ref, name):
    _report(name, got, ref)
    assert got.shape == ref.shape and torch.equal(got.view(torch.int16), ref.view(torch.int16)), f"{name}: not bit-identical"


# ======================================================================================================================
# A. pixel-strip temporal attention
# ======================================================================================================================
def _strip(S, world, k):
    """Pixels [s0, s1) that rank k computes: strips ceil(S / world) wide, the last ones short or empty."""
    per = -(-S // world)
    return min(k * per, S), min((k + 1) * per, S)


@pytest.mark.parametrize("B,Tl,world,S,heads", [
    pytest.param(2, 1, 16, 37, 1, id="w16-Tl1-S37"),
    pytest.param(1, 2, 8, 64, 5, id="w8-Tl2-S64-h5"),
    pytest.param(2, 4, 4, 10, 10, id="w4-Tl4-S10-h10"),
    pytest.param(1, 8, 2, 33, 5, id="w2-Tl8-S33-h5"),
    pytest.param(2, 3, 5, 23, 1, id="w5-Tl3-T15-S23"),
    pytest.param(1, 1, 16, 5, 5, id="w16-Tl1-S5-empty-strips"),
    pytest.param(2, 2, 8, 3, 10, id="w8-Tl2-S3-empty-strips"),
    pytest.param(1, 1, 2, 1, 1, id="w2-Tl1-S1"),
    pytest.param(1, 16, 1, 20, 2, id="w1-Tl16"),
    pytest.param(2, 8, 2, 4096, 5, id="bench-w2-Tl8-S4096-h5"),
    pytest.param(2, 8, 2, 16384, 5, id="bench-w2-Tl8-S16384-h5"),
])
def test_sharded_temporal_attention(B, Tl, world, S, heads):
    Cc, T = heads * 64, Tl * world
    qkv = [rnd(B * Tl * S, 3 * Cc, seed=100 + r).to(H) for r in range(world)]
    outs = [_nans(B * Tl * S, Cc) for _ in range(world)]
    Q, O = _World(qkv), _World(outs)

    # ownership: launched alone, rank k fills pixel strip k of EVERY rank's output and nothing else
    for k in range(world):
        for o in outs:
            o.fill_(NAN)
        ops.temporal_attention_d64_sharded(Q, O, k, world, B, Tl, S, heads)
        s0, s1 = _strip(S, world, k)
        mine = torch.zeros(S, dtype=torch.bool, device=DEV)
        mine[s0:s1] = True
        for r, o in enumerate(outs):
            nan = torch.isnan(o.view(B, Tl, S, Cc))
            assert not bool(nan[:, :, mine].any()), f"rank {k} left rows of its strip [{s0}, {s1}) in rank {r}'s output unset"
            assert bool(nan[:, :, ~mine].all()), f"rank {k} wrote rows outside its strip [{s0}, {s1}) in rank {r}'s output"

    for o in outs:
        o.fill_(NAN)
    for k in range(world):
        ops.temporal_attention_d64_sharded(Q, O, k, world, B, Tl, S, heads)
    # gather: rank r's frames go to frame slots [r Tl, (r+1) Tl) of every clip
    full_qkv = torch.cat([q.view(B, Tl, S, 3 * Cc) for q in qkv], 1).reshape(B * T * S, 3 * Cc)
    got = torch.cat([o.view(B, Tl, S, Cc) for o in outs], 1).reshape(B * T * S, Cc)

    q, k_, v = (t.view(B, T, S, heads, 64).permute(0, 2, 3, 1, 4).float() for t in full_qkv.view(-1, 3, Cc).unbind(1))
    ref = torch.softmax(q @ k_.transpose(-1, -2) * 0.125, -1) @ v
    _check(got.view(B, T, S, heads, 64).permute(0, 2, 3, 1, 4), ref, f"sharded temporal attention x{world} vs fp32", atol=2e-3)

    # each (clip, pixel, head) item does the same arithmetic whichever rank computes it
    unsharded = torch.zeros(B * T * S, Cc, dtype=H, device=DEV)
    ops.temporal_attention_d64(full_qkv, B, T, S, heads, unsharded)
    _identical(got, unsharded, f"sharded temporal attention x{world} vs unsharded kernel")


# ======================================================================================================================
# B. temporal GroupNorm: all-reduced statistics, haloed output, halo frames stored into the neighbours' buffers
# ======================================================================================================================
class _GnWorld:
    """x_r [B * Tl * HW, C] per rank, and the haloed GroupNorm outputs gh_r [B * (Tl + 2) * HW, C] (NaN before each apply).

    Routes to the statistics, as unet._Plan takes them in peer mode (`_resblock_impl`):
      "unit"  -- hi3d_groupnorm_unit_stats per rank (the table a producing GEMM epilogue accumulates), then
                 hi3d_groupnorm_group_sums(imgs_per_sample = Tl), summed over ranks, hi3d_groupnorm_apply_halo;
      "stats" -- hi3d_groupnorm_apply_stats with neighbour pointers, reading the ranks' unit tables laid side by side as one
                 [B, T, units] table (imgs_per_sample = T)."""

    def __init__(self, B, Tl, world, Cc, HW, mean=0.0, seed=0):
        self.B, self.Tl, self.world, self.C, self.HW, self.T = B, Tl, world, Cc, HW, Tl * world
        offs = mean + 0.1 * rnd(Cc, seed=seed + 90)          # a per-channel offset around the mean
        self.x = [(rnd(B * Tl * HW, Cc, seed=seed + r) * 0.5 + offs).to(H) for r in range(world)]
        self.gamma, self.beta = 1 + 0.1 * rnd(Cc, seed=seed + 91), 0.1 * rnd(Cc, seed=seed + 92)
        self.gh = [_nans(B * (Tl + 2) * HW, Cc) for _ in range(world)]

    def _nbr(self, r):
        prev = self.gh[r - 1].data_ptr() if r > 0 else None
        nxt = self.gh[r + 1].data_ptr() if r + 1 < self.world else None
        return prev, nxt

    def statistics(self, route):
        """What the apply launches read: the all-reduced sums [B, 32, 2], or for route "stats" the gathered unit table.
        (The statistics kernels add with float atomics, so two passes may differ in the last bit: compute them once.)"""
        assert route in ("unit", "stats"), route
        B, Tl, HW, Cc = self.B, self.Tl, self.HW, self.C
        tables = []
        for x in self.x:
            t = torch.zeros(B * Tl, Cc // GN_UNIT, 2, device=DEV)
            ops.groupnorm_unit_stats(x, B * Tl, HW, GN_UNIT, t.view(-1))
            tables.append(t)
        if route == "stats":
            return torch.cat([t.view(B, Tl, -1, 2) for t in tables], 1).contiguous()
        local = []
        for r in range(self.world):
            s = torch.zeros(B, 32, 2, device=DEV)
            ops.groupnorm_group_sums(tables[r].view(-1), Cc, None, 0, GN_UNIT, B, Tl, s)
            local.append(s)
        total = torch.zeros(B, 32, 2, device=DEV)
        for s in local:                                       # the exchange kernel's all-reduce: rank order
            total = total + s
        return total

    def apply(self, route, stats, silu, order):
        B, Tl, HW, T = self.B, self.Tl, self.HW, self.T
        for g in self.gh:
            g.fill_(NAN)
        for r in order:
            prev, nxt = self._nbr(r)
            if route == "stats":
                ops.groupnorm_apply_stats(self.x[r], stats.view(-1), None, None, GN_UNIT, B, Tl * HW, T, T * HW, self.gamma,
                                          self.beta, 1e-5, silu, self.gh[r], (Tl + 2) * HW, HW, y_prev=prev, y_next=nxt,
                                          frame_rows=HW)
            else:
                ops.groupnorm_apply(self.x[r], None, B, Tl * HW, stats, T * HW, self.gamma, self.beta, 1e-5, silu, self.gh[r],
                                    y_sample_rows=(Tl + 2) * HW, y_row_off=HW, y_prev=prev, y_next=nxt, frame_rows=HW)

    def frames(self, r):
        return self.gh[r].view(self.B, self.Tl + 2, self.HW, self.C)

    def interior(self):
        """The gathered normalised clip [B, T, HW, C]: frames 1 .. Tl of every rank's haloed buffer."""
        return torch.cat([self.frames(r)[:, 1:self.Tl + 1] for r in range(self.world)], 1)

    def reference(self, silu):
        B, T, HW, Cc = self.B, self.T, self.HW, self.C
        xf = torch.cat([x.view(B, self.Tl, HW, Cc) for x in self.x], 1).float().view(B, T * HW, Cc).permute(0, 2, 1)
        ref = F.group_norm(xf, 32, self.gamma, self.beta, 1e-5)
        if silu:
            ref = F.silu(ref)
        return ref.permute(0, 2, 1).reshape(B, T, HW, Cc)

    def check_halos(self, name):
        """Leading slot of rank r = rank r-1's last frame, trailing slot = rank r+1's first frame, bit for bit; at the clip
        boundaries the slot is exactly zero (it was NaN before the launch)."""
        Tl, W = self.Tl, self.world
        for r in range(W):
            v = self.frames(r)
            lead, trail = v[:, 0], v[:, Tl + 1]
            if r == 0:
                assert bool((lead.view(torch.int16) == 0).all()), f"{name}: rank 0's leading halo slot is not zero-filled"
            else:
                _identical(lead, self.frames(r - 1)[:, Tl], f"{name}: rank {r} leading halo slot")
            if r == W - 1:
                assert bool((trail.view(torch.int16) == 0).all()), f"{name}: rank {r}'s trailing halo slot is not zero-filled"
            else:
                _identical(trail, self.frames(r + 1)[:, 1], f"{name}: rank {r} trailing halo slot")


GN_CASES = [
    pytest.param(1, 16, 320, 64, True, 0.0, id="Tl1-w16-c320-hw64"),
    pytest.param(2, 8, 640, 64, False, 0.0, id="Tl2-w8-c640-hw64-nosilu"),
    pytest.param(4, 4, 1280, 1024, True, 0.0, id="Tl4-w4-c1280-hw1024"),
    pytest.param(8, 2, 320, 4096, True, 0.0, id="Tl8-w2-c320-hw4096"),
    pytest.param(8, 2, 640, 1024, False, 0.0, id="Tl8-w2-c640-hw1024-nosilu"),
    pytest.param(8, 2, 1280, 64, True, 0.0, id="Tl8-w2-c1280-hw64"),
    pytest.param(2, 8, 320, 1024, True, 2.0, id="Tl2-w8-c320-hw1024-mean4std"),
    pytest.param(3, 5, 320, 100, True, 0.0, id="Tl3-w5-c320-hw100"),
]


@pytest.mark.parametrize("route", ["unit", "stats"])
@pytest.mark.parametrize("Tl,world,Cc,HW,silu,mean", GN_CASES)
def test_sharded_temporal_groupnorm_halo(Tl, world, Cc, HW, silu, mean, route):
    gw = _GnWorld(2, Tl, world, Cc, HW, mean=mean, seed=7)
    name = f"GN {route} x{world}"
    stats = gw.statistics(route)
    gw.apply(route, stats, silu, range(world))
    _check(gw.interior(), gw.reference(silu), f"{name} interior vs fp32 F.group_norm")
    gw.check_halos(f"{name} ascending")
    first = [g.clone() for g in gw.gh]
    # launch order does not matter: no rank's launch overwrites a slot another rank stored
    gw.apply(route, stats, silu, range(world - 1, -1, -1))
    gw.check_halos(f"{name} descending")
    for r in range(world):
        _identical(gw.gh[r], first[r], f"{name} rank {r}: descending vs ascending launch order")


# ======================================================================================================================
# C. (3,1,1) temporal conv over the haloed buffers, both engines
# ======================================================================================================================
@pytest.fixture
def pair_mode():
    lib = _native.load()

    def set_(m):
        _native.check(lib.hi3d_gemm_tc5_set_pair_mode(m), "set_pair_mode")
    yield set_
    set_(-1)


def _tc5_tiles(Tl, HW, N):
    """The wgmma engine's temporal tiling rule (hi3d_gemm_tc5): ts pixels x 128 / ts frames per tile, else mma.sync."""
    ts = 1
    while ts * 2 <= 128 and HW % (ts * 2) == 0:
        ts *= 2
    return N >= 32 and N % 8 == 0 and Tl % (128 // ts) == 0


@pytest.mark.parametrize("engine,pair", [("mma", -1), ("tc5", -1), ("tc5", 0), ("tc5", 1)],
                         ids=["mma", "tc5-auto", "tc5-single", "tc5-pairs"])
@pytest.mark.parametrize("path,B,Tl,world,HW,Cc", [
    pytest.param("tc5", 2, 8, 2, 4096, 320, id="tc5tiles-Tl8-hw4096-c320"),
    pytest.param("tc5", 2, 8, 2, 1024, 640, id="tc5tiles-autopairs-Tl8-hw1024-c640"),
    pytest.param("tc5", 2, 8, 2, 64, 1280, id="tc5tiles-2frames-per-tile-Tl8-hw64-c1280"),
    pytest.param("tc5", 1, 8, 2, 48, 320, id="tc5tiles-3tiles-Tl8-hw48-c320"),
    pytest.param("mma", 2, 1, 16, 64, 320, id="tc5-forwards-to-mma-Tl1-hw64-c320"),
    pytest.param("mma", 2, 4, 4, 16, 640, id="tc5-forwards-to-mma-Tl4-hw16-c640"),
    pytest.param("mma", 2, 3, 5, 100, 320, id="tc5-forwards-to-mma-Tl3-hw100-c320"),
])
def test_sharded_temporal_conv_over_halo_then_unit_stats(pair_mode, engine, pair, path, B, Tl, world, HW, Cc):
    assert _tc5_tiles(Tl, HW, Cc) == (path == "tc5"), "case id names the wrong engine path"
    pair_mode(pair)
    gw = _GnWorld(B, Tl, world, Cc, HW, seed=11)
    gw.apply("unit", gw.statistics("unit"), True, range(world))
    T, M = Tl * world, B * Tl * HW
    interior = gw.interior()
    _check(interior, gw.reference(True), "conv source interior vs fp32 F.group_norm")

    w = rnd(Cc, Cc, 3, 1, 1, scale=(3 * Cc) ** -0.5, seed=12)
    wp = pack.pack_conv3d_t(w)
    bias = rnd(Cc, scale=0.1, seed=13)
    emb = rnd(B, T, Cc, scale=0.5, seed=14).to(H)                 # per-frame embedding row
    xs = rnd(B, T, HW, Cc, seed=15).to(H)                          # residual / blend source
    alpha = 0.3
    xr = interior.permute(0, 3, 1, 2).unsqueeze(-1).float()        # [B, C, T, HW, 1]
    conv = F.conv3d(xr, w.to(H).float(), bias, padding=(1, 0, 0)).squeeze(-1).permute(0, 2, 3, 1)   # [B, T, HW, Co]
    geo = dict(Ho=HW, Wo=1, T=Tl, Tin=Tl + 2, t_off=1)
    tag = f"{engine} pair={pair} x{world}"
    for r in range(world):
        sl = slice(r * Tl, (r + 1) * Tl)
        cr = conv[:, sl].reshape(M, Cc)
        # 1. bias + per-frame rowbias (the temporal ResBlock's first conv)
        out = _nans(M, Cc)
        st = torch.zeros(B * Tl, Cc // GN_UNIT, 2, device=DEV)
        ops.Gemm(ops.temporal_taps(gw.gh[r]), wp, out, M, mode=ops.ROWS_TEMPORAL, geom=geo, bias=bias,
                 rowbias=emb[:, sl].reshape(B * Tl, Cc), rb_div=HW, rb_mod=B * Tl, engine=engine)()
        ops.groupnorm_unit_stats(out, B * Tl, HW, GN_UNIT, st.view(-1))
        ref = cr + emb[:, sl].float().repeat_interleave(HW, 1).reshape(M, Cc)
        _check(out, ref, f"temporal conv + rowbias rank {r} {tag}")
        _close_stats(st, _unit_sums(out, B * Tl, HW, GN_UNIT), f"unit stats rank {r} {tag}")
        # 2. bias + residual + alpha blend (the second conv: out = alpha x + (1 - alpha) (x + conv))
        res = xs[:, sl].reshape(M, Cc)
        out = _nans(M, Cc)
        st = torch.zeros(B * Tl, Cc // GN_UNIT, 2, device=DEV)
        ops.Gemm(ops.temporal_taps(gw.gh[r]), wp, out, M, mode=ops.ROWS_TEMPORAL, geom=geo, bias=bias, residual=res,
                 blend_x=res, alpha=alpha, engine=engine)()
        ops.groupnorm_unit_stats(out, B * Tl, HW, GN_UNIT, st.view(-1))
        ref = alpha * res.float() + (1 - alpha) * (cr.to(H).float() + res.float())
        _check(out, ref, f"temporal conv + residual + blend rank {r} {tag}")
        _close_stats(st, _unit_sums(out, B * Tl, HW, GN_UNIT), f"unit stats (blend) rank {r} {tag}")


# ======================================================================================================================
# D. exchange kernel, rank 0 only, with nothing to wait for
# ======================================================================================================================
# Word layout of one rank's exchange area (csrc/peer.cu): [0, 64) flags, then payload[parity][rank][1024], then the local
# epoch counter 32 words into the 256-byte tail.
XCHG_FLAGS, XCHG_SLOT = 64, 1024


def _epoch_word(world):
    return XCHG_FLAGS + 2 * world * XCHG_SLOT + 32


def _slot(area, world, par, r, n):
    base = XCHG_FLAGS + (par * world + r) * XCHG_SLOT
    return area[base:base + n].view(torch.float32)


def _xchg_areas(world):
    nbytes = int(_native.load().hi3d_peer_xchg_bytes(world))
    assert nbytes >= 4 * (_epoch_word(world) + 1)
    areas = [torch.zeros(nbytes // 4, dtype=torch.int32, device=DEV) for _ in range(world)]
    return areas, (C.c_void_p * world)(*[a.data_ptr() for a in areas])


def _exchange_rank0(areas, ptrs, world, payload, n, out):
    """One exchange as rank 0.  Every flag word rank 0 could wait on is preset to 2^30 first, so for any epoch this test
    reaches the kernel finds every rank already past it: a misread layout shows as a wrong value, never as a wait."""
    areas[0][:XCHG_FLAGS] = 2 ** 30
    torch.cuda.synchronize()
    rc = _native.load().hi3d_peer_exchange(ptrs, 0, world, payload.data_ptr(), n, out.data_ptr(), _stream())
    torch.cuda.synchronize()
    return rc


def _bits(t):
    return t.contiguous().view(torch.int32)


@pytest.mark.parametrize("n", [0, 1, 64, 1024])
def test_exchange_single_rank(n):
    areas, ptrs = _xchg_areas(1)
    ew = _epoch_word(1)
    for call in range(1, 4):
        payload = rnd(max(n, 1), seed=200 + call)
        out = torch.full((max(n, 1),), NAN, device=DEV)
        assert _exchange_rank0(areas, ptrs, 1, payload, n, out) == 0
        assert int(areas[0][ew]) == call, f"epoch word {int(areas[0][ew])} after call {call}"
        if n == 0:
            assert bool(torch.isnan(out).all()), "an exchange without payload wrote its output"
        else:
            exp = torch.zeros(n, device=DEV) + payload[:n]
            _report(f"exchange x1 n={n} call {call}", out[:n], exp)
            assert torch.equal(_bits(out[:n]), _bits(exp))


@pytest.mark.parametrize("world", [2, 4, 16])
def test_exchange_sums_in_rank_order(world):
    n = 1000
    areas, ptrs = _xchg_areas(world)
    ew = _epoch_word(world)
    # the simulated peers' payloads, different in the two parity halves (reading the wrong half shows) and of mixed
    # magnitudes (summing in another order rounds differently)
    peer = {(par, r): rnd(n, scale=10.0 ** (r % 4 - 1), seed=300 + 17 * r + par) for par in (0, 1) for r in range(1, world)}
    for (par, r), v in peer.items():
        _slot(areas[0], world, par, r, n).copy_(v)
    torch.cuda.synchronize()
    prev = torch.zeros(n, device=DEV)
    for e in range(1, 4):
        par = e & 1
        p0 = rnd(n, seed=400 + e)
        out = torch.full((n,), NAN, device=DEV)
        assert _exchange_rank0(areas, ptrs, world, p0, n, out) == 0
        assert int(areas[0][ew]) == e, f"epoch word {int(areas[0][ew])} after call {e}"
        exp = torch.zeros(n, device=DEV)
        for r in range(world):
            exp = exp + (p0 if r == 0 else peer[par, r])
        _report(f"exchange x{world} call {e}", out, exp)
        assert torch.equal(_bits(out), _bits(exp)), f"call {e}: not the float32 sum in rank order of parity half {par}"
        for r in range(1, world):
            a = areas[r]
            assert int(a[0]) == e, f"rank {r}: flag word 0 = {int(a[0])}, expected epoch {e}"
            assert bool((a[1:XCHG_FLAGS] == 0).all()), f"rank {r}: flag words other than rank 0's were written"
            assert int(a[ew]) == 0, f"rank {r}: its local epoch word was written"
            assert torch.equal(_bits(_slot(a, world, par, 0, n)), _bits(p0)), f"rank {r}: payload not in slot [{par}][0]"
            assert torch.equal(_bits(_slot(a, world, 1 - par, 0, n)), _bits(prev)), \
                f"rank {r}: slot [{1 - par}][0] changed, the parity did not alternate"
        prev = p0


# ======================================================================================================================
# E. argument rejection, with real buffers sized for the geometry requested
# ======================================================================================================================
def _all_nan(*ts):
    torch.cuda.synchronize()
    return all(bool(torch.isnan(t).all()) for t in ts)


@pytest.mark.parametrize("world,Tl", [(4, 5), (2, 9), (17, 1)])
def test_rejects_sharded_attention_past_16_frames(world, Tl):
    B, S, heads = 1, 8, 1
    qkv = [rnd(B * Tl * S, 3 * 64, seed=r).to(H) for r in range(world)]
    outs = [_nans(B * Tl * S, 64) for _ in range(world)]
    Q, O = _World(qkv), _World(outs)
    rc = _native.load().hi3d_temporal_attention_d64_sharded(Q.ptr_array, O.ptr_array, 0, world, B, Tl, S, heads, 0.125,
                                                            _stream())
    assert rc == -2
    assert _all_nan(*outs)


def test_rejects_groupnorm_halo_geometry():
    lib = _native.load()
    B, Tl, HW, Cc = 2, 2, 64, 320
    rows = Tl * HW
    x = rnd(B * rows, Cc, seed=1).to(H)
    gam, bet = 1 + 0.1 * rnd(Cc, seed=2), 0.1 * rnd(Cc, seed=3)
    table = torch.zeros(B * Tl, Cc // GN_UNIT, 2, device=DEV)
    ops.groupnorm_unit_stats(x, B * Tl, HW, GN_UNIT, table.view(-1))
    sums = torch.zeros(B, 32, 2, device=DEV)
    ops.groupnorm_group_sums(table.view(-1), Cc, None, 0, GN_UNIT, B, Tl, sums)
    cap = B * (Tl + 4) * HW               # room for every store the requested geometry could address
    y, yp, yn = _nans(cap, Cc), _nans(cap, Cc), _nans(cap, Cc)
    bad = [((Tl + 3) * HW, HW, HW),       # y_sample_rows != rows + 2 frame_rows
           ((Tl + 1) * HW, HW, HW),
           ((Tl + 2) * HW, 2 * HW, HW),   # y_row_off != frame_rows
           ((Tl + 2) * HW, 0, HW),
           (rows + 96, 48, 48)]           # frame_rows does not divide the rows
    for ysr, off, fr in bad:
        for prev, nxt in ((yp, yn), (None, yn), (yp, None), (None, None)):
            pp, np_ = (None if prev is None else prev.data_ptr()), (None if nxt is None else nxt.data_ptr())
            rc = lib.hi3d_groupnorm_apply_halo(x.data_ptr(), Cc, None, 0, B, rows, sums.data_ptr(), 2 * rows, gam.data_ptr(),
                                               bet.data_ptr(), 1e-5, 1, y.data_ptr(), ysr, off, pp, np_, fr, _stream())
            assert rc == -2, (ysr, off, fr)
            rc = lib.hi3d_groupnorm_apply_stats(x.data_ptr(), Cc, table.data_ptr(), None, 0, None, GN_UNIT, B, rows, Tl, rows,
                                                gam.data_ptr(), bet.data_ptr(), 1e-5, 1, y.data_ptr(), ysr, off, pp, np_, fr,
                                                _stream())
            assert rc == -2, (ysr, off, fr)
    assert _all_nan(y, yp, yn)


@pytest.mark.parametrize("engine", ["mma", "tc5"])
def test_rejects_temporal_conv_past_source_frames(engine):
    B, Tl, HW, Cc = 1, 8, 16, 64
    src = rnd(B * (Tl + 2) * HW, Cc, seed=1).to(H)      # a real haloed source, Tin = Tl + 2 frames per clip
    wp = pack.pack_conv3d_t(rnd(Cc, Cc, 3, 1, 1, scale=(3 * Cc) ** -0.5, seed=2))
    out = _nans(B * Tl * HW, Cc)
    fn = _native.load().hi3d_gemm_tc5 if engine == "tc5" else _native.load().hi3d_gemm
    for tin, t_off in ((Tl + 2, 3), (Tl + 2, Tl + 2), (Tl + 1, 2), (Tl - 1, 0)):      # t_off + T > Tin
        g = ops.Gemm(ops.temporal_taps(src), wp, out, B * Tl * HW, mode=ops.ROWS_TEMPORAL,
                     geom=dict(Ho=HW, Wo=1, T=Tl, Tin=tin, t_off=t_off), engine=engine)
        assert fn(C.byref(g.p), _stream()) == -2, (tin, t_off)
    assert _all_nan(out)


def test_rejects_exchange_payload_over_1024():
    areas, ptrs = _xchg_areas(1)
    n = 1025
    payload, out = rnd(n, seed=5), torch.full((n,), NAN, device=DEV)
    assert _exchange_rank0(areas, ptrs, 1, payload, n, out) == -2
    assert _all_nan(out)
    assert int(areas[0][_epoch_word(1)]) == 0
