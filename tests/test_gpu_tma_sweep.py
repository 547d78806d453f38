"""Every width and pipeline shape of the TMA conv and weight-gradient kernels (csrc/nn_conv_tma.cu), bit for bit against
float64.

Integer operands make these kernels exactly checkable: activation codes 0..15, odd weight codes -15..15 and gradients in
-8..8 are exact in bf16, every product and partial sum is an integer below 2^24, so the fp32 accumulation is exact in any
order, and a power-of-two code scale adds no rounding.  The float64 reference (rounded to integers first, so that the
algorithm torch picks cannot matter) times the fp32 scale, rounded to fp32 once, is then bit-identical to what a correct
kernel stores: any wrong tap, chunk, column, row half, ring stage, split or fragment register is a mismatch.  The noisy
output adds z * sigma with sigma = sqrt.approx(coef * S): with raw weights on a 1/8 grid, g(|w|) is exact in bf16 and S
is exact, so the only rounding left is a few ulp of the MUFU square root and the final multiply-add.

Every GPU case runs under torch.profiler and asserts which instantiation launched (k_conv_tma<EPI, NT>,
k_wgrad_tma<TAIL, TW>): the routing falls back to the gathered kernels without a word when a call is not served.  The
expected NT, stage count and weight-gradient split come from a restatement of the plans (tma_plan / wgrad_plan below),
which the CPU tests pin against the library's nn_weight_pack_bytes and against the instantiations in the source.
"""
import ctypes as C
import os
import re

import numpy as np
import pytest
import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
TMA_SRC = os.path.join(ROOT, "noisynet_b200", "csrc", "nn_conv_tma.cu")

S_A, S_W = 0.25, 0.125          # power-of-two code scales: a scaled integer sum is exact in fp32
NOISE_SCALE, CURRENT = 0.75, 1.5
SMS_H100 = 132                  # H100 SXM; the GPU tests use the device's own count
NONE, MERGED, EXTERNAL = 0, 1, 2


# ---------------------------------------------------------------------------------------------- plan restatements

def _pad(v, a):
    return (v + a - 1) // a * a


def _cdiv(a, b):
    return -(-a // b)


def tma_plan(cin_k, k, n_out, sigma):
    """nn_tma_make_plan (csrc/nn_conv_tma.cu) for a k x k filter over cin_k channels producing n_out columns (+ the
    sigma^2 columns when noisy); None where the plan refuses.  The forward passes (Cin, k, Cout), the dgrad (Cout, k, Cin)."""
    Cp = _pad(cin_k, 8)
    if Cp <= 8:
        return None
    taps = k * k
    n_c64 = Cp // 64
    rem = Cp - 64 * n_c64
    tail_w = 0 if rem == 0 else 16 if rem <= 16 else 32 if rem <= 32 else 64
    nc = n_c64 + (1 if tail_w else 0)
    wt = 64 * n_c64 + tail_w
    gpt = (nc + 1) // 2
    max_nt = 120 if sigma else 256
    n_tiles = _cdiv(n_out, max_nt)
    n_t = _pad(_cdiv(n_out, n_tiles), 8)
    n_tiles = _cdiv(n_out, n_t)
    n_mma = max(32, _pad(2 * n_t if sigma else n_t, 16))
    if n_mma > 256:
        return None
    gw = 0                                  # widest group of two channel chunks
    for gi in range(gpt):
        ca, cb = 2 * gi, 2 * gi + 1
        wa = 64 if ca < n_c64 else tail_w
        wb = (64 if cb < n_c64 else tail_w) if cb < nc else 0
        gw = max(gw, wa + wb)
    stage = _pad(256 * gw, 1024) + _pad(n_mma * 2 * gw, 1024)
    stages = min(8, (222 * 1024 - 2048) // stage)
    if stages < 2:
        return None
    tap_bytes = 2 * (n_mma // 2) * 2 * wt
    return dict(n_t=n_t, n_tiles=n_tiles, n_mma=n_mma, stages=stages, n_groups=taps * gpt, tail_w=tail_w,
                wp_bytes=n_tiles * taps * tap_bytes)


def wgrad_plan(cin, k, cout, mpix, sms=SMS_H100):
    """nn_tma_wgrad_plan plus the launch choices of nn_tma_wgrad_launch and the reduce's group counts (nn_conv_umma.cu)."""
    Cp = _pad(cin, 8)
    n_c64, tail = Cp // 64, Cp % 64
    if n_c64 == 0:
        return None
    taps = k * k
    if tail > 8 or (tail == 8 and taps > 31):       # wider remainders (and > 31 taps): one more zero-filled chunk
        n_c64, tail = n_c64 + 1, 0
    n_atoms = taps * n_c64
    tiles_k = _cdiv(n_atoms, 4)
    num_kb = _cdiv(mpix, 64)
    splits = max(1, min(sms // (tiles_k * _cdiv(cout, 128)), num_kb))
    kb_per_split = _cdiv(num_kb, splits)
    splits = _cdiv(num_kb, kb_per_split)

    def groups(quads, cnt):
        g = 1
        while g < 32 and quads * g < 131072 and cnt >= 8 * g:
            g *= 2
        return g

    return dict(widths={64 * min(4, n_atoms - 4 * t) for t in range(tiles_k)}, tw=_pad(taps * 8, 16) if tail else 0,
                splits=splits, kb_per_split=kb_per_split, g_main=groups(cout * tiles_k * 64, splits),
                g_tail=groups(cout * 64, splits) if tail else 1)


def conv_name(epi, nt):
    return "k_conv_tma<%d, %d>" % (epi, nt)


def wgrad_names(wp):
    return {"k_wgrad_tma<false, 0>", "k_wgrad_tma_reduce"} | ({"k_wgrad_tma<true, %d>" % wp["tw"]} if wp["tw"] else set())


# ---------------------------------------------------------------------------------------------- GPU cases
# forward: (B, Cin, H, Cout, k, stride, pad) with square images
PLAIN_NT = list(range(8, 257, 8))
NOISY_COUT = list(range(8, 121, 8)) + [121, 200, 240, 241, 256, 390, 512]


def plain_cases(nt):
    """Cout = NT over a 64 + 16-channel tail and over two 64-channel chunks; every other width also ragged (NT - 3):
    B * OH * OW = 300 pixels, three m-tiles (the odd last pair)."""
    couts = [nt] + ([nt - 3] if (nt // 8) % 2 == 0 else [])
    return [(3, cin, 12, cout, 3, 1, 0) for cin in (65, 128) for cout in couts]


def noisy_case(cout):
    return (3, 65 if cout % 16 else 128, 12, cout, 3, 1, 0)


def dgrad_case(nt):
    """layer (B, Cin, H, Cout, k, pad): the dgrad's n-tile is the layer's Cin (NT, or 8 k + 1 padded to NT), its channels
    the layer's Cout (16: tail only, 65: chunk + tail, 128: two chunks), k = 1..5 and pads 0..k-1"""
    i = nt // 8 - 1
    k = 1 + i % 5
    return (3, nt if i % 2 == 0 else nt - 7, 10, (16, 65, 128)[i % 3], k, (i // 5) % k)


GEOMETRY = [  # B, Cin, H, Cout, k, stride, pad
    (2, 72, 9, 40, 2, 1, 0),            # even filter: wgrad remainder width 32, dgrad pad 1
    (2, 72, 10, 24, 4, 1, 1),           # 4x4: wgrad remainder width 128
    (2, 65, 11, 48, 6, 1, 2),           # 6x6: 36 taps, the wgrad remainder as a zero-filled chunk
    (2, 136, 7, 40, 4, 1, 2),           # 128 + 8 channels, 4x4: remainder at channel 128
    (2, 65, 13, 56, 3, 2, 1),           # stride 2 (forward and wgrad only)
    (2, 128, 14, 64, 3, 3, 0),          # stride 3
    (1, 72, 23, 16, 7, 2, 3),           # 7x7 stride 2 pad 3: 49 taps, zero-filled remainder chunk
    (2, 96, 10, 136, 1, 2, 0),          # 1x1 stride 2, 64 + 32 channels, two n-tiles when noisy
]

WGRAD = [  # B, Cin, H, Cout, k, stride, pad
    (2, 72, 9, 24, 1, 1, 0),            # remainder widths 16 / 32 / 80 / 128 / 208 at channel 64 ...
    (2, 72, 9, 40, 2, 1, 1),
    (2, 72, 10, 24, 3, 2, 1),
    (2, 72, 9, 16, 4, 1, 2),
    (2, 72, 9, 24, 5, 1, 2),
    (2, 136, 7, 16, 1, 2, 0),           # ... and at channel 128
    (2, 136, 7, 24, 2, 1, 0),
    (2, 136, 8, 16, 3, 1, 1),
    (1, 136, 8, 40, 4, 1, 1),
    (1, 136, 9, 16, 5, 1, 2),
    (2, 64, 9, 24, 1, 1, 0),            # last column tile of 1 .. 4 atoms
    (2, 128, 9, 40, 1, 1, 0),
    (2, 192, 9, 24, 1, 1, 0),
    (2, 64, 9, 40, 2, 1, 0),
    (2, 64, 9, 24, 3, 1, 1),            # 9 atoms: tiles of 4, 4, 1
    (3, 72, 9, 200, 3, 1, 1),           # Cout > 128, ragged
    (2, 64, 8, 390, 1, 1, 0),
    (1, 72, 8, 24, 3, 1, 1),            # 64 pixels: one k-block in all
    (3, 65, 14, 120, 5, 1, 0),          # conv2, 300 pixels: one k-block per split
    (64, 64, 12, 16, 1, 1, 0),          # 144 k-blocks over 72 splits: reduce groups G = 8
    (40, 72, 12, 16, 3, 1, 1),          # 90 k-blocks over 30 splits: remainder groups G = 2
]

# persistent runs: >= 3 pairs per co-resident cluster, an odd m-tile count, n_groups % stages != 0 (the ring phase runs
# on across items); kind, B, Cin, H, Cout, k, pad  (the dgrad rows give the layer's geometry)
MULTI = [
    ("noisy", 354, 120, 12, 104, 3, 1),    # S = 2
    ("plain", 354, 65, 13, 236, 2, 0),     # S = 3
    ("dgrad", 354, 233, 12, 40, 3, 1),     # S = 4
    ("noisy", 354, 40, 12, 100, 3, 1),     # S = 5
    ("plain", 354, 40, 12, 136, 3, 1),     # S = 6
    ("dgrad", 354, 81, 12, 40, 3, 1),      # S = 7
    ("noisy", 354, 16, 12, 60, 3, 1),      # S = 8
]


def multi_plan(case):
    kind, B, cin, H, cout, k, pad = case
    if kind == "dgrad":
        return tma_plan(cout, k, cin, False), B * H * H
    OH = H + 2 * pad - k + 1
    return tma_plan(cin, k, cout, kind == "noisy"), B * OH * OH


# ---------------------------------------------------------------------------------------------- CPU tests

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from noisynet_b200 import _lib
    return _lib.load()


def test_plan_restatement_matches_pack_bytes(lib):
    """tma_plan's image size equals the library's for forward (plain / noisy) and dgrad NN_PACK_TMA jobs"""
    from noisynet_b200._lib import PACK_TMA, WPrepJob
    n = 0
    for cin in (9, 16, 24, 33, 40, 64, 65, 72, 96, 120, 128, 136, 200, 256):
        for k in (1, 2, 3, 4, 5, 7):
            for cout in (1, 8, 13, 64, 120, 121, 200, 233, 256, 390, 512):
                for mode, noise in ((0, NONE), (0, EXTERNAL), (0, MERGED), (1, NONE)):
                    jb = WPrepJob()
                    jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.noise_mode, jb.layout = cout, cin, k * k, mode, noise, PACK_TMA
                    p = tma_plan(cin, k, cout, noise != NONE) if mode == 0 else tma_plan(cout, k, cin, False)
                    want = _pad(p["wp_bytes"], 1024) if p else 0
                    assert lib.nn_weight_pack_bytes(C.byref(jb)) == want, (cin, k, cout, mode, noise, p)
                    n += want > 0
    assert n > 1000


def _instantiated():
    """the k_conv_tma / k_wgrad_tma instantiations of the source"""
    src = open(TMA_SRC).read()
    conv = set()
    for epi, lo, hi in re.findall(r"tma_conv_kernel<(\d), (\d+), (\d+)>\(pl\.n_t\)", src):
        conv |= {(int(epi), nt) for nt in range(int(lo), int(hi) + 1, 8)}
    tails = {int(t) for t in re.findall(r"k_wgrad_tma<true, (\d+)>", src)}
    return conv, tails


def _covered():
    conv, widths, tails = set(), set(), set()
    for nt in PLAIN_NT:
        for B, cin, H, cout, k, s, p in plain_cases(nt):
            conv.add((2, tma_plan(cin, k, cout, False)["n_t"]))
        B, cin, H, cout, k, p = dgrad_case(nt)
        conv.add((2, tma_plan(cout, k, cin, False)["n_t"]))
    for cout in NOISY_COUT:
        B, cin, H, cout, k, s, p = noisy_case(cout)
        conv |= {(1, tma_plan(cin, k, cout, True)["n_t"]), (3, tma_plan(cin, k, cout, True)["n_t"])}
    for B, cin, H, cout, k, s, p in GEOMETRY + WGRAD:
        OH = (H + 2 * p - k) // s + 1
        wp = wgrad_plan(cin, k, cout, B * OH * OH)
        widths |= wp["widths"]
        tails.add(wp["tw"])
    return conv, widths, tails


def test_sweep_covers_every_instantiation():
    conv_src, tails_src = _instantiated()
    assert len(conv_src) == 32 + 15 + 15 and max(nt for e, nt in conv_src if e != 2) == 120
    conv, widths, tails = _covered()
    assert conv == conv_src, conv_src ^ conv
    assert widths == {64, 128, 192, 256}
    assert tails - {0} == tails_src == {16, 32, 80, 128, 208}
    wps = [wgrad_plan(cin, k, cout, B * ((H + 2 * p - k) // s + 1) ** 2) for B, cin, H, cout, k, s, p in WGRAD]
    assert any(w["kb_per_split"] == 1 and w["splits"] > 1 for w in wps)
    assert any(w["g_main"] > 1 for w in wps) and any(w["g_tail"] > 1 for w in wps)
    # zero-filled remainder chunks (6x6, 7x7 with 8 remainder channels)
    assert any(_pad(cin, 8) % 64 == 8 and k * k > 31 for B, cin, H, cout, k, s, p in GEOMETRY)
    # persistent runs: every ring depth, the phase running on across items, the odd last pair, >= 3 pairs per cluster
    stages = set()
    for case in MULTI:
        pl, m = multi_plan(case)
        n_mt = _cdiv(m, 128)
        assert pl["n_groups"] % pl["stages"] and n_mt % 2 == 1, case
        assert (n_mt + 1) // 2 * pl["n_tiles"] >= 3 * (SMS_H100 // 2), case
        stages.add(pl["stages"])
    assert stages == set(range(2, 9))
    assert {c[0] for c in MULTI} == {"noisy", "plain", "dgrad"}


# ---------------------------------------------------------------------------------------------- exact oracle

def _exact(t):
    """a float64 evaluation of an integer contraction -> its integers (each value must already be one)"""
    r = torch.round(t)
    assert (r - t).abs().max().item() <= 1e-6
    assert r.abs().max().item() < 2 ** 24
    return r


def _scaled(r, scale):
    """what the kernels store for the integer sums r: ONE fp32 multiply by the fp32 scale, rounded to nearest"""
    return r.float() * torch.tensor(float(np.float32(scale)), dtype=torch.float32, device=r.device)


def test_exact_oracle_detects_one_off():
    gen = torch.Generator().manual_seed(3)
    ka, cw = _act_codes((2, 65, 9, 9), gen), _w_codes((24, 65, 3, 3), gen)
    want = _scaled(_exact(F.conv2d(ka.double(), cw.double())), S_A * S_W)
    got = F.conv2d(ka, cw) * (S_A * S_W)          # fp32 over exact integers: the same bits
    assert torch.equal(got, want)
    bad = _exact(F.conv2d(ka.double(), cw.double()))
    bad[1, 7, 3, 4] += 1
    assert not torch.equal(got, _scaled(bad, S_A * S_W))
    with pytest.raises(AssertionError):
        _exact(F.conv2d(ka.double(), cw.double()) + 0.5 * (torch.rand(want.shape, generator=gen) > 0.99).double())
    # noisy: the few-ulp bound takes the reference and rejects one ulp-scale error of 1e-5 relative
    z = torch.randn(want.shape, generator=gen)
    ref, tol = _noisy_ref(want, torch.ones_like(want, dtype=torch.float64), z, _coef())
    out = ref.float()
    _assert_within(out, ref, tol)
    out[0, 0, 0, 0] += 1e-5 * max(1.0, abs(out[0, 0, 0, 0].item()))
    with pytest.raises(AssertionError):
        _assert_within(out, ref, tol)


def _act_codes(shape, gen):
    k = torch.randint(0, 16, shape, generator=gen).float()
    return k * (torch.rand(shape, generator=gen) > 0.25).float()


def _w_codes(shape, gen):
    return (torch.randint(0, 16, shape, generator=gen) * 2 - 15).float()


def _w_raw(shape, gen):
    """raw weights j / 8, 0 < |j| <= 8: g(|w|) is exact in bf16 (and no value sits on a rounding tie of the 4-bit
    quantizer of [-1, 1])"""
    j = torch.randint(1, 9, shape, generator=gen) * (torch.randint(0, 2, shape, generator=gen) * 2 - 1)
    return j.float() / 8.0


def _grads(shape, gen):
    return torch.randint(-8, 9, shape, generator=gen).float()


def _coef():
    """nn_noise_coef: 0.1 * (scale / current), both fp32 roundings"""
    return float(np.float32(0.1) * (np.float32(NOISE_SCALE) / np.float32(CURRENT)))


def _sigma_sum(ka, w_raw, mode, stride, pad):
    """S = conv(activation codes, g(|w|)) in float64, exact: 64 g(|w|) is an integer on the 1/8 grid"""
    a = w_raw.double().abs()
    g = a if mode == MERGED else a * a + a
    return _exact(F.conv2d(ka.double(), g * 64.0, None, stride, pad)) / 64.0


def _noisy_ref(y, s, z, coef):
    """y_noisy = y + z * sqrt(coef * S * s_a) in float64, and the bound of a correct kernel: a few ulp of the noise
    term (sqrt.approx, the fp32 rounding of coef * S and of z * sigma) plus the final rounding"""
    noise = z.double().to(y.device) * torch.sqrt(coef * (s * S_A))
    ref = y.double() + noise
    return ref, 2.0 ** -21 * noise.abs() + 2.0 ** -22 * ref.abs() + 1e-30


def _assert_within(out, ref, tol):
    d = (out.double().to(ref.device) - ref).abs()
    bad = d > tol
    assert not bool(bad.any()), "%d values off, worst %.3e (bound %.3e) at %s" % (
        int(bad.sum()), (d - tol).max().item(), tol.flatten()[int((d - tol).argmax())].item(),
        np.unravel_index(int((d - tol).argmax()), tuple(d.shape)))


# ---------------------------------------------------------------------------------------------- GPU plumbing

@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


_KERNEL = re.compile(r"\b(k_conv_tma|k_wgrad_tma_reduce|k_wgrad_tma|k_conv_umma|k_wgrad_umma|k_splitk_epilogue|"
                     r"k_wgrad_umma_reduce2?|k_conv_shift|k_wgrad_shift)\b(<[^>]*>)?")


def _launch(expect, fn, exact=True):
    """runs fn under torch.profiler; the conv / wgrad kernels it launched must be exactly `expect` (exact=False: include
    these kernel names, whatever their template arguments, and no TMA kernel)"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        out = fn()
        torch.cuda.synchronize()
    seen = set()
    for e in prof.events():
        m = _KERNEL.search(e.name)
        if m:
            seen.add(m.group(1) + (m.group(2) or ""))
    from noisynet_b200 import ops
    assert ops.error_flag() == 0
    if exact:
        assert seen == set(expect), (sorted(seen), sorted(expect))
    else:
        assert set(expect) <= {n.split("<")[0] for n in seen} and not any("_tma" in n for n in seen), (sorted(seen), sorted(expect))
    return out


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _scale_dev(dev):
    return torch.tensor([NOISE_SCALE], device=dev)


def _fwd_plain(dev, ka, cw, stride, pad, expect, s_a=S_A, s_w=S_W):
    from noisynet_b200 import ops
    x, w = (ka * np.float32(s_a)).to(dev), (cw * np.float32(s_w)).to(dev)
    return _launch(expect, lambda: ops.noisy_conv_fwd(x, w, None, None, stride, pad, precision="bf16", a_code_scale=s_a,
                                                      w_code_scale=s_w)["y"])


def _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, expect, **kw):
    from noisynet_b200 import ops
    x, w = (ka * S_A).to(dev), (cw * S_W).to(dev)
    return _launch(expect, lambda: ops.noisy_conv_fwd(
        x, w, wr.to(dev), None, stride, pad, noise_mode=mode, current=CURRENT, scale_dev=_scale_dev(dev), precision="bf16",
        a_code_scale=S_A, w_code_scale=S_W, want_y=False, **kw)["y_noisy"])


def _z_fp32(dev, ka, cw, wr, stride, pad, mode, rng):
    """the Philox draws of (rng) as the fp32 CUDA-core kernel exports them"""
    from noisynet_b200 import ops
    return ops.noisy_conv_fwd((ka * S_A).to(dev), (cw * S_W).to(dev), wr.to(dev), None, stride, pad, noise_mode=mode,
                              current=CURRENT, scale_dev=_scale_dev(dev), precision="fp32", rng=rng, want_z=True)["z"]


def check_noisy(dev, ka, cw, wr, stride, pad, mode, nt, y_int, on, gen, repeat=False):
    """<3, NT> with injected draws against the oracle; <1, NT> (Philox) against <3, NT> fed the fp32 kernel's draws"""
    from noisynet_b200 import ops
    s = _sigma_sum(ka.to(on), wr.to(on), mode, stride, pad)
    y = _scaled(y_int, S_A * S_W).double()
    z = torch.randn(tuple(y.shape), generator=gen)
    out = _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, {conv_name(3, nt)}, z=z.to(dev))
    _assert_within(out, *_noisy_ref(y, s, z, _coef()))
    rng = ops._fixed_rng(1234 + nt, 7)
    o1 = _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, {conv_name(1, nt)}, rng=rng)
    z32 = _z_fp32(dev, ka, cw, wr, stride, pad, mode, rng)
    o3 = _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, {conv_name(3, nt)}, z=z32)
    ref, tol = _noisy_ref(y, s, z32, _coef())
    _assert_within(o3, ref, tol)
    _assert_within(o1, o3.double().to(ref.device), tol)
    if repeat:
        assert torch.equal(o1, _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, {conv_name(1, nt)}, rng=rng))
        assert torch.equal(o3, _fwd_noisy(dev, ka, cw, wr, stride, pad, mode, {conv_name(3, nt)}, z=z32))


def _dgrad(dev, gy, cw, x_shape, pad, expect, s_w=S_W):
    from noisynet_b200 import ops
    g, w = gy.to(dev), (cw * np.float32(s_w)).to(dev)
    return _launch(expect, lambda: ops.conv_dgrad(g, w, x_shape, 1, pad, precision="bf16", w_code_scale=s_w))


def _wgrad(dev, gy, ka, w_shape, stride, pad, expect, **kw):
    from noisynet_b200 import ops
    g, x = gy.to(dev), (ka * S_A).to(dev)
    return _launch(expect, lambda: ops.conv_wgrad(g, x, w_shape, stride, pad, precision="bf16", a_code_scale=S_A, **kw))


def check_wgrad(dev, ka, gy, w_shape, stride, pad, on, gen, repeat=False):
    B, Cin, H, _ = ka.shape
    Cout, _, k, _ = w_shape
    wp = wgrad_plan(Cin, k, Cout, gy.shape[0] * gy.shape[2] * gy.shape[3], _sms())
    want = _scaled(_exact(torch.nn.grad.conv2d_weight(ka.to(on).double(), w_shape, gy.to(on).double(), stride, pad)), S_A)
    gw = _wgrad(dev, gy, ka, w_shape, stride, pad, wgrad_names(wp))
    assert torch.equal(gw.to(on), want)
    w_raw = torch.randn(w_shape, generator=gen)
    gwm = _wgrad(dev, gy, ka, w_shape, stride, pad, wgrad_names(wp), w_raw=w_raw.to(dev), w_lo=-1.0, w_hi=1.0)
    keep = ((w_raw >= -1.0) & (w_raw <= 1.0)).to(on)
    assert torch.equal(gwm.to(on), torch.where(keep, want, torch.zeros_like(want)))
    if repeat:
        assert torch.equal(gw, _wgrad(dev, gy, ka, w_shape, stride, pad, wgrad_names(wp)))


# ---------------------------------------------------------------------------------------------- GPU tests

@pytest.mark.gpu
@pytest.mark.parametrize("nt", PLAIN_NT)
def test_forward_plain_width(dev, nt):
    gen = torch.Generator().manual_seed(nt)
    for B, cin, H, cout, k, s, p in plain_cases(nt):
        assert tma_plan(cin, k, cout, False)["n_t"] == nt
        ka, cw = _act_codes((B, cin, H, H), gen), _w_codes((cout, cin, k, k), gen)
        r = _exact(F.conv2d(ka.double(), cw.double(), None, s, p))
        y = _fwd_plain(dev, ka, cw, s, p, {conv_name(2, nt)})
        assert torch.equal(y.cpu(), _scaled(r, S_A * S_W)), (cin, cout)
        if nt in (8, 120, 256) and cout == nt:
            # the real 4-bit scales 5/15, 1/15: one fp32 multiply by fp32(fp32(5/15) * fp32(1/15))
            y = _fwd_plain(dev, ka, cw, s, p, {conv_name(2, nt)}, s_a=5.0 / 15.0, s_w=1.0 / 15.0)
            assert torch.equal(y.cpu(), _scaled(r, np.float32(5.0 / 15.0) * np.float32(1.0 / 15.0)))
            exact = r * (float(np.float32(5.0 / 15.0)) * float(np.float32(1.0 / 15.0)))
            assert torch.allclose(y.cpu().double(), exact, rtol=1e-6, atol=1e-9)


@pytest.mark.gpu
@pytest.mark.parametrize("cout", NOISY_COUT)
def test_forward_noisy_width(dev, cout):
    B, cin, H, cout, k, s, p = noisy_case(cout)
    nt = tma_plan(cin, k, cout, True)["n_t"]
    gen = torch.Generator().manual_seed(100 + cout)
    ka, cw, wr = _act_codes((B, cin, H, H), gen), _w_codes((cout, cin, k, k), gen), _w_raw((cout, cin, k, k), gen)
    y_int = _exact(F.conv2d(ka.double(), cw.double(), None, s, p))
    for mode in (EXTERNAL, MERGED):
        check_noisy(dev, ka, cw, wr, s, p, mode, nt, y_int, torch.device("cpu"), gen)


@pytest.mark.gpu
@pytest.mark.parametrize("nt", PLAIN_NT)
def test_dgrad_width(dev, nt):
    B, cin, H, cout, k, p = dgrad_case(nt)
    assert tma_plan(cout, k, cin, False)["n_t"] == nt
    gen = torch.Generator().manual_seed(300 + nt)
    OH = H + 2 * p - k + 1
    cw, gy = _w_codes((cout, cin, k, k), gen), _grads((B, cout, OH, OH), gen)
    gx = _dgrad(dev, gy, cw, (B, cin, H, H), p, {conv_name(2, nt)})
    r = _exact(torch.nn.grad.conv2d_input((B, cin, H, H), cw.double(), gy.double(), 1, p))
    assert torch.equal(gx.cpu(), _scaled(r, S_W))


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GEOMETRY)
def test_geometry(dev, shape):
    B, cin, H, cout, k, s, p = shape
    cpu = torch.device("cpu")
    gen = torch.Generator().manual_seed(sum(shape))
    ka, cw, wr = _act_codes((B, cin, H, H), gen), _w_codes((cout, cin, k, k), gen), _w_raw((cout, cin, k, k), gen)
    y_int = _exact(F.conv2d(ka.double(), cw.double(), None, s, p))
    y = _fwd_plain(dev, ka, cw, s, p, {conv_name(2, tma_plan(cin, k, cout, False)["n_t"])})
    assert torch.equal(y.cpu(), _scaled(y_int, S_A * S_W))
    check_noisy(dev, ka, cw, wr, s, p, EXTERNAL, tma_plan(cin, k, cout, True)["n_t"], y_int, cpu, gen)
    gy = _grads(tuple(y_int.shape), gen)
    if s == 1:
        gx = _dgrad(dev, gy, cw, (B, cin, H, H), p, {conv_name(2, tma_plan(cout, k, cin, False)["n_t"])})
        r = _exact(torch.nn.grad.conv2d_input((B, cin, H, H), cw.double(), gy.double(), 1, p))
        assert torch.equal(gx.cpu(), _scaled(r, S_W))
    check_wgrad(dev, ka, gy, (cout, cin, k, k), s, p, cpu, gen)


@pytest.mark.gpu
@pytest.mark.parametrize("shape", WGRAD)
def test_wgrad(dev, shape):
    B, cin, H, cout, k, s, p = shape
    gen = torch.Generator().manual_seed(500 + sum(shape))
    OH = (H + 2 * p - k) // s + 1
    ka, gy = _act_codes((B, cin, H, H), gen), _grads((B, cout, OH, OH), gen)
    check_wgrad(dev, ka, gy, (cout, cin, k, k), s, p, torch.device("cpu"), gen)


@pytest.mark.gpu
@pytest.mark.parametrize("case", MULTI, ids=lambda c: "%s-%d-%d-%d" % (c[0], c[2], c[4], c[5]))
def test_persistent_multi_item(dev, case):
    """many items per cluster: whole tensors against float64 (on the GPU), and a second launch bit-identical"""
    kind, B, cin, H, cout, k, pad = case
    pl, m = multi_plan(case)
    assert (_cdiv(m, 128) + 1) // 2 * pl["n_tiles"] >= 3 * (_sms() // 2)
    gen = torch.Generator().manual_seed(700 + cin + cout)
    nt = pl["n_t"]
    if kind == "dgrad":
        cw, gy = _w_codes((cout, cin, k, k), gen), _grads((B, cout, H, H), gen)
        r = _exact(torch.nn.grad.conv2d_input((B, cin, H, H), cw.to(dev).double(), gy.to(dev).double(), 1, pad))
        gxs = [_dgrad(dev, gy, cw, (B, cin, H, H), pad, {conv_name(2, nt)}) for _ in range(2)]
        assert torch.equal(gxs[0], _scaled(r, S_W))
        assert torch.equal(gxs[0], gxs[1])
        return
    ka, cw = _act_codes((B, cin, H, H), gen), _w_codes((cout, cin, k, k), gen)
    y_int = _exact(F.conv2d(ka.to(dev).double(), cw.to(dev).double(), None, 1, pad))
    if kind == "plain":
        ys = [_fwd_plain(dev, ka, cw, 1, pad, {conv_name(2, nt)}) for _ in range(2)]
        assert torch.equal(ys[0], _scaled(y_int, S_A * S_W))
        assert torch.equal(ys[0], ys[1])
    else:
        wr = _w_raw((cout, cin, k, k), gen)
        check_noisy(dev, ka, cw, wr, 1, pad, EXTERNAL, nt, y_int, dev, gen, repeat=True)


@pytest.mark.gpu
def test_conv2_batch512_forward(dev):
    """NoisyNet conv2 at batch 512: <1, 120> and <3, 120>, whole tensors, EXTERNAL noise as the training step runs it"""
    gen = torch.Generator().manual_seed(512)
    ka, cw, wr = _act_codes((512, 65, 14, 14), gen), _w_codes((120, 65, 5, 5), gen), _w_raw((120, 65, 5, 5), gen)
    y_int = _exact(F.conv2d(ka.to(dev).double(), cw.to(dev).double()))
    check_noisy(dev, ka, cw, wr, 1, 0, EXTERNAL, 120, y_int, dev, gen, repeat=True)


@pytest.mark.gpu
def test_conv2_batch512_dgrad(dev):
    gen = torch.Generator().manual_seed(513)
    cw, gy = _w_codes((120, 65, 5, 5), gen), _grads((512, 120, 10, 10), gen)
    r = _exact(torch.nn.grad.conv2d_input((512, 65, 14, 14), cw.to(dev).double(), gy.to(dev).double()))
    gxs = [_dgrad(dev, gy, cw, (512, 65, 14, 14), 0, {conv_name(2, 72)}) for _ in range(2)]
    assert torch.equal(gxs[0], _scaled(r, S_W))
    assert torch.equal(gxs[0], gxs[1])


@pytest.mark.gpu
def test_conv2_batch512_wgrad(dev):
    """~45 k-blocks per split: the 4-stage ring wraps ~11 times; the full tensor, with and without the STE mask"""
    gen = torch.Generator().manual_seed(514)
    ka, gy = _act_codes((512, 65, 14, 14), gen), _grads((512, 120, 10, 10), gen)
    wp = wgrad_plan(65, 5, 120, 51200, _sms())
    assert wp["kb_per_split"] >= 40 and wp["tw"] == 208
    check_wgrad(dev, ka, gy, (120, 65, 5, 5), 1, 0, dev, gen, repeat=True)


def _nhwc_bf16(t, cp):
    """the packed activation / grad-output image: [B][H][W][Cp] bf16, channels past C zero (DESIGN.md section 3)"""
    B, Cn, H, W = t.shape
    out = torch.zeros(B, H, W, cp, dtype=torch.bfloat16, device=t.device)
    out[..., :Cn] = t.permute(0, 2, 3, 1).to(torch.bfloat16)
    return out


@pytest.mark.gpu
def test_packed_operands_conv2(dev):
    """conv2's NN_PACK_TMA forward (noisy) and dgrad images from nn_prepare_weights (4-bit quantizer, round to nearest,
    as the engine fills its jobs), and NHWC bf16 activation / grad-output images, through the C ABI"""
    from noisynet_b200 import _lib, ops
    from noisynet_b200._lib import (PACK_TMA, PREC_BF16, ConvDgradArgs, ConvFwdArgs, ConvGeom, ConvWgradArgs, Rng,
                                    WPrepJob)
    from oracle import noisynet_oracle as O
    lib = _lib.load()
    B, Cin, H, Cout, k = 6, 65, 14, 120, 5
    OH = H - k + 1
    gen = torch.Generator().manual_seed(65)
    wr = _w_raw((Cout, Cin, k, k), gen)
    ka, gy = _act_codes((B, Cin, H, H), gen), _grads((B, Cout, OH, OH), gen)
    w_cs = float(np.float32(2.0 / 15.0)) / 2.0
    wq = O.uniform_quantize_fwd(wr, 4, -1.0, 1.0)
    codes = torch.round(wq.double() / w_cs)
    assert (codes - wq.double() / w_cs).abs().max().item() < 1e-4 and bool((codes.remainder(2) == 1).all())
    geom = ConvGeom(B, Cin, H, H, Cout, k, k, 1, 0)
    assert lib.nn_conv_pack_layout(C.byref(geom), EXTERNAL, PREC_BF16) == PACK_TMA
    assert lib.nn_conv_dgrad_pack_layout(C.byref(geom), PREC_BF16) == PACK_TMA
    wr_d = wr.to(dev)
    jobs = (WPrepJob * 2)()
    code_scratch = torch.zeros(wr.numel() + 16, dtype=torch.int8, device=dev)
    bufs = []
    for j, (mode, noise) in enumerate(((0, EXTERNAL), (1, NONE))):
        jb = jobs[j]
        jb.w_raw = wr_d.data_ptr()
        jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows, jb.noise_mode, jb.want_wsum = Cout, Cin, k * k, mode, B * OH * OH, noise, 0
        jb.layout, jb.q_bits, jb.q_hi, jb.stochastic, jb.u_inject, jb.rng = PACK_TMA, 4, 1.0, 0.0, None, Rng(0, 0, None)
        jb.codes = code_scratch.data_ptr()
        buf = torch.zeros(int(lib.nn_weight_pack_bytes(C.byref(jb))) + 1024, dtype=torch.uint8, device=dev)
        jb.packed_out = (buf.data_ptr() + 1023) // 1024 * 1024
        bufs.append(buf)
    st = torch.cuda.current_stream().cuda_stream
    _lib.check(lib.nn_prepare_weights(jobs, 2, 0, st), "nn_prepare_weights")
    xp, gyp = _nhwc_bf16(ka.to(dev), 72), _nhwc_bf16(gy.to(dev), 120)
    ws = torch.empty(int(max(lib.nn_conv_workspace_bytes(C.byref(geom), PREC_BF16),
                             lib.nn_conv_wgrad_workspace_bytes(C.byref(geom), PREC_BF16, 0))) + 4096, dtype=torch.uint8, device=dev)
    z = torch.randn(B, Cout, OH, OH, generator=gen).to(dev)
    scale = _scale_dev(dev)

    # forward: packed weights and activations, injected draws -> <3, 120>
    yn = torch.empty(B, Cout, OH, OH, device=dev)
    a = ConvFwdArgs()
    a.g, a.w_raw, a.y_noisy, a.noise_mode, a.current, a.scale_dev = geom, None, yn.data_ptr(), EXTERNAL, CURRENT, scale.data_ptr()
    a.z_inject, a.rng, a.precision, a.a_code_scale, a.w_code_scale = z.data_ptr(), Rng(0, 0, None), PREC_BF16, S_A, w_cs
    a.workspace, a.workspace_bytes = ws.data_ptr(), ws.numel()
    a.x_packed, a.w_packed, a.w_packed_layout = xp.data_ptr(), jobs[0].packed_out, PACK_TMA
    _launch({conv_name(3, 120)}, lambda: _lib.check(lib.nn_noisy_conv_fwd(C.byref(a), 0, st), "nn_noisy_conv_fwd"))
    y_int = _exact(F.conv2d(ka.double(), codes))
    y = _scaled(y_int, np.float32(S_A) * np.float32(w_cs)).double()
    _assert_within(yn, *_noisy_ref(y, _sigma_sum(ka, wr, EXTERNAL, 1, 0), z.cpu(), _coef()))
    ref_call = ops.noisy_conv_fwd((ka * S_A).to(dev), (codes.float() * w_cs).to(dev), wr_d, None, 1, 0, noise_mode=EXTERNAL,
                                  current=CURRENT, scale_dev=scale, z=z, precision="bf16", a_code_scale=S_A,
                                  w_code_scale=w_cs, want_y=False)["y_noisy"]
    assert torch.equal(yn, ref_call)

    # dgrad: packed dgrad image and grad-output -> <2, 72>
    gx = torch.empty(B, Cin, H, H, device=dev)
    d = ConvDgradArgs()
    d.g, d.gy, d.w_eff, d.gx, d.precision, d.w_code_scale = geom, None, None, gx.data_ptr(), PREC_BF16, w_cs
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    d.gy_packed, d.w_packed, d.w_packed_layout = gyp.data_ptr(), jobs[1].packed_out, PACK_TMA
    _launch({conv_name(2, 72)}, lambda: _lib.check(lib.nn_noisy_conv_dgrad(C.byref(d), 0, st), "nn_noisy_conv_dgrad"))
    r = _exact(torch.nn.grad.conv2d_input((B, Cin, H, H), codes, gy.double()))
    assert torch.equal(gx.cpu(), _scaled(r, w_cs))
    assert torch.equal(gx, ops.conv_dgrad(gy.to(dev), (codes.float() * w_cs).to(dev), (B, Cin, H, H), 1, 0, precision="bf16",
                                          w_code_scale=w_cs))

    # weight gradient: packed activations and grad-output ([pixel][Coutp] = the same NHWC image)
    wp = wgrad_plan(Cin, k, Cout, B * OH * OH, _sms())
    gw = torch.empty(Cout, Cin, k, k, device=dev)
    g = ConvWgradArgs()
    g.g, g.gy, g.x, g.gw, g.precision, g.a_code_scale = geom, None, None, gw.data_ptr(), PREC_BF16, S_A
    g.workspace, g.workspace_bytes = ws.data_ptr(), ws.numel()
    g.x_packed, g.gy_packed, g.gy_packed_layout = xp.data_ptr(), gyp.data_ptr(), 0
    _launch(wgrad_names(wp), lambda: _lib.check(lib.nn_noisy_conv_wgrad(C.byref(g), 0, st), "nn_noisy_conv_wgrad"))
    r = _exact(torch.nn.grad.conv2d_weight(ka.double(), (Cout, Cin, k, k), gy.double()))
    assert torch.equal(gw.cpu(), _scaled(r, S_A))
    assert torch.equal(gw, ops.conv_wgrad(gy.to(dev), (ka * S_A).to(dev), (Cout, Cin, k, k), precision="bf16", a_code_scale=S_A))
    assert ops.error_flag() == 0


GATHERED = [  # B, Cin, H, Cout, k, stride, pad
    (3, 65, 14, 120, 5, 1, 0),
    (3, 128, 12, 256, 3, 1, 1),
    (2, 72, 9, 24, 5, 1, 2),
    (2, 136, 7, 40, 4, 1, 2),
]


@pytest.mark.gpu
@pytest.mark.parametrize("shape", GATHERED)
def test_gathered_kernels_exact(dev, shape):
    """the same exact oracle for the gathered-im2col kernels (TMA paths switched off)"""
    from noisynet_b200 import _lib, ops
    B, cin, H, cout, k, s, p = shape
    gen = torch.Generator().manual_seed(900 + sum(shape))
    ka, cw = _act_codes((B, cin, H, H), gen), _w_codes((cout, cin, k, k), gen)
    y_int = _exact(F.conv2d(ka.double(), cw.double(), None, s, p))
    gy = _grads(tuple(y_int.shape), gen)
    x, w, g = (ka * S_A).to(dev), (cw * S_W).to(dev), gy.to(dev)
    lib = _lib.load()
    prev = lib.nn_debug_tma_enable(0)
    try:
        y = _launch({"k_conv_umma"}, lambda: ops.noisy_conv_fwd(x, w, None, None, s, p, precision="bf16", a_code_scale=S_A,
                                                                 w_code_scale=S_W)["y"], exact=False)
        gx = _launch({"k_conv_umma"}, lambda: ops.conv_dgrad(g, w, (B, cin, H, H), 1, p, precision="bf16", w_code_scale=S_W),
                     exact=False)
        gw = _launch({"k_wgrad_umma"}, lambda: ops.conv_wgrad(g, x, (cout, cin, k, k), s, p, precision="bf16", a_code_scale=S_A),
                     exact=False)
    finally:
        lib.nn_debug_tma_enable(prev)
    assert torch.equal(y.cpu(), _scaled(y_int, S_A * S_W))
    assert torch.equal(gx.cpu(), _scaled(_exact(torch.nn.grad.conv2d_input((B, cin, H, H), cw.double(), gy.double(), 1, p)), S_W))
    assert torch.equal(gw.cpu(), _scaled(_exact(torch.nn.grad.conv2d_weight(ka.double(), (cout, cin, k, k), gy.double(), s, p)), S_A))
