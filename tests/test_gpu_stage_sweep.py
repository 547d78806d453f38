"""The between-layer stage kernels (csrc/nn_stage.cu: pool, BatchNorm, ReLU, clamp, quantize, pack and their backward)
against float64 and exact fp32 restatements, at the training step's shapes and batch sizes.

The batch statistics are split over batch slices (stage_splits: one per 2048 elements of a channel, at most 16), so the
step's shapes at batch 512 run 16 slices (65 x 14 x 14), 6 slices (120 x 5 x 5) and 1 slice (390); batches 500, 777 and
1024 split B unevenly.  The operands are chosen so that the checks can be exact:

- Forward inputs are multiples of 1/4 in [-4, 4]: 2x2 windows have tied maxima (the first in row-major order must win,
  as in nn.MaxPool2d), and every per-slice sum and sum of squares is exact in double, so the partial sums left in the
  scratch are checked bit for bit, which pins the slice count, the slice bounds and the scratch layout.
- gamma is a signed power of two, so fl(xhat * gamma) is exact and an FMA contraction of xhat * gamma + beta gives the
  same v as two roundings: the codes are restated in numpy float32 from the kernel's own mean / invstd and must match
  bit for bit (Philox draws from oracle.philox4x32_10, groups 2i and 2i + 1 of thread i = pixel * Cp/8 + chunk).
- Backward operands are built from v on a 1/4 grid (dyadic mean, power-of-two invstd and gamma), so v lands exactly on
  0, on act_max and on q_hi (pinning > against >=), and dbeta / dgamma are exact sums.

Every GPU case runs under torch.profiler and asserts which instantiations launched; the expected ones come from the
restatements of nn_stage_fwd / nn_stage_bwd's dispatch below, which the CPU tests pin against the library and the source.
The dropout (<true>) instantiations are covered by test_gpu_dropout.py.
"""
import ctypes as C
import os
import re
import time

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
STAGE_SRC = os.path.join(ROOT, "noisynet_b200", "csrc", "nn_stage.cu")

ST_SPLITS = 16                  # most batch slices per channel
ST_REC = ST_SPLITS * 2 + 2      # doubles per channel record of the scratch: partials, then the counter padded to 16 bytes
EPS, MOM = np.float32(1e-5), np.float32(0.1)
ACT_MAX, BITS, Q_HI, STOCH = 5.0, 4, 4.0, 0.5
QMAX = np.float32(2 ** BITS - 1)
Q_SCALE = np.float32(Q_HI / (2 ** BITS - 1))
SEED, OFFSET = 0x5EED1234ABCD, 77


def _pad8(c):
    return (c + 7) // 8 * 8


# ---------------------------------------------------------------------------------------------- dispatch restatements

def stage_splits(per_channel):
    """stage_splits: one slice per 2048 elements of a channel, 1 .. ST_SPLITS"""
    return max(1, min(ST_SPLITS, per_channel // 2048))


def slice_bounds(B, splits):
    """samples [b0, b1) of each slice: b0 = B * s / splits (integer division)"""
    return [(B * s // splits, B * (s + 1) // splits) for s in range(splits)]


def scratch_bytes(C_):
    """nn_stage_scratch_bytes: C channel records of ST_REC doubles (channel c's record at byte c * 8 * ST_REC: slice s's
    sum and sum of squares at doubles 2s, 2s + 1, the arrival counter at double 2 * ST_SPLITS)"""
    return C_ * ST_REC * 8


def fwd_kernels(B, C_, H, W, pool, stats_ready=False, act=False, u_inject=False, stoch=STOCH):
    """the kernels nn_stage_fwd launches (quantised; no dropout)"""
    HW = (H // 2) * (W // 2) if pool else H * W
    Cp = _pad8(C_)
    ks = set() if stats_ready else {"k_pool_stats" if pool else "k_chan_stats"}
    items = B * HW * Cp // 8
    lean = stoch > 0 and not u_inject and not act and B * C_ * HW < 2 ** 31 and items < 2 ** 31
    if lean and HW >= 32 and 32 * ((Cp // 8) | 1) * 16 <= 48 * 1024:
        ks.add("k_bn_act_pack_tiled<false>")
    elif lean:
        ks.add("k_bn_act_pack_lean<false>")
    else:
        ks.add("k_bn_act_pack<false>")
    return ks


def bwd_kernels(B, C_, H, W, pool, planes, f32):
    """the kernels nn_stage_bwd launches (no dropout); H, W of the stage input"""
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    Cp = _pad8(C_)
    items = B * PH * PW * Cp // 8
    lean = not f32 and B * C_ * PH * PW < 2 ** 31 and items < 2 ** 31
    if lean and pool and not planes and H * W * Cp * 2 <= 48 * 1024 and PH * PW >= 16:
        apply = "k_bn_bwd_apply_img<false>"
    elif not lean:
        apply = "k_bn_bwd_apply<false>"
    else:
        apply = "k_bn_bwd_apply_lean<%s, %s, false>" % ("true" if pool else "false", "true" if planes else "false")
    return {"k_bn_bwd_stats<false>", apply}


# (B, C, H, W, pool, stats_ready): the step's stage shapes (65 x 14 x 14 also as the fused conv1 path calls it, statistics
# ready; and without pooling: k_chan_stats over 16 slices), batches that split B unevenly, batch 1024
FWD = [(512, 65, 28, 28, 1, 0), (500, 65, 28, 28, 1, 0), (1024, 65, 28, 28, 1, 0), (512, 65, 14, 14, 0, 1),
       (777, 65, 14, 14, 0, 0), (512, 120, 10, 10, 1, 0), (777, 120, 10, 10, 1, 0), (1024, 120, 10, 10, 1, 0),
       (512, 390, 1, 1, 0, 0)]
# (B, C, H, W, pool, planes): bn1's backward into conv1's wgrad planes (32 x 32 grid), pooled NHWC, bn2's per-image
# kernel, bn3, and an unpooled planes output
BWD = [(512, 65, 28, 28, 1, 1), (500, 65, 28, 28, 1, 0), (512, 120, 10, 10, 1, 0), (777, 120, 10, 10, 1, 0),
       (1024, 120, 10, 10, 1, 0), (512, 390, 1, 1, 0, 0), (512, 65, 14, 14, 0, 1)]
PLANES_GRID = {28: (32, 32), 14: (16, 16)}


def _source_instantiations():
    """the stage kernels nn_stage_fwd / nn_stage_bwd launch in the source, without the dropout (<true>) ones"""
    src = open(STAGE_SRC).read()
    body = src[src.index('extern "C" int nn_stage_fwd'):src.index("// ---", src.index('extern "C" int nn_stage_bwd'))]
    names = {n + (t or "") for n, t in re.findall(r"\b(k_\w+)(<[^>]*>)?<<<", body)}
    return {n for n in names if not n.endswith("true>")}


def test_dispatch_covers_every_instantiation():
    got = set()
    for B, C_, H, W, pool, ready in FWD:
        got |= fwd_kernels(B, C_, H, W, pool, ready) | fwd_kernels(B, C_, H, W, pool, ready, act=True)
    for B, C_, H, W, pool, planes in BWD:
        got |= bwd_kernels(B, C_, H, W, pool, planes, False) | bwd_kernels(B, C_, H, W, pool, planes, True)
    src = _source_instantiations()
    assert len(src) == 12
    assert got == src, got ^ src


def test_step_shapes_split_as_stated():
    """the slice counts the step runs at batch 512, and uneven slices at the other batches"""
    assert [stage_splits(512 * hw) for hw in (196, 25, 1)] == [16, 6, 1]
    assert stage_splits(768 * 25) == 9 and stage_splits(737 * 25) == 8 and stage_splits(1024 * 25) == 12
    for B, C_, H, W, pool, _ in FWD:
        hw = (H // 2) * (W // 2) if pool else H * W
        s = stage_splits(B * hw)
        sizes = {b1 - b0 for b0, b1 in slice_bounds(B, s)}
        assert sum(b1 - b0 for b0, b1 in slice_bounds(B, s)) == B
        if B in (500, 777):
            assert len(sizes) == 2, (B, s)


@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from noisynet_b200 import _lib
    return _lib.load()


def test_scratch_layout_matches_library(lib):
    """per-channel records: channel c's counter sits at the same byte whatever the calling stage's C (the GPU tests read
    the partial sums and counters back at these offsets)"""
    for c in range(1, 1025):
        assert lib.nn_stage_scratch_bytes(c) == scratch_bytes(c), c


# ---------------------------------------------------------------------------------------------- references

def _philox_u(B, C_, HW, seed=SEED, offset=OFFSET, stoch=STOCH):
    """the stochastic-rounding draws of thread i = pixel * Cp/8 + chunk: channel c reads group 2i + (c % 8) / 4, word
    c % 4; u = fl(fl(u01(r) * fl(2s)) - s).  [B, C, HW] float32"""
    from oracle.noisynet_oracle import philox4x32_10
    chunks = _pad8(C_) // 8
    i = np.arange(B * HW * chunks, dtype=np.uint64)
    g = np.stack([2 * i, 2 * i + 1], axis=-1)                             # [threads, 2]
    r = philox4x32_10(g, seed, offset).reshape(B * HW, chunks * 8)[:, :C_]
    u01 = (r >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24)
    u = (u01 * np.float32(2.0 * stoch)).astype(np.float32) - np.float32(stoch)
    return np.ascontiguousarray(u.reshape(B, HW, C_).transpose(0, 2, 1))


def _v(x, mean, invstd, gamma, beta, fma=False):
    """fl(fl(fl(x - mean) * invstd) * gamma + beta), per channel (axis 1 of [B, C, HW]); exact for power-of-two gamma
    whether or not the kernel contracts the last two operations into an FMA.  fma=True: the contracted form
    fl(xhat * gamma + beta) with one rounding (the product is exact in float64)"""
    e = lambda a: a.astype(np.float32)[None, :, None]
    xhat = ((x - e(mean)) * e(invstd)).astype(np.float32)
    if fma:
        return xhat, (xhat.astype(np.float64) * e(gamma).astype(np.float64) + e(beta).astype(np.float64)).astype(np.float32)
    return xhat, (xhat * e(gamma) + e(beta)).astype(np.float32)


def _codes(x, mean, invstd, gamma, beta, u, act_max=ACT_MAX, q_scale=Q_SCALE, qmax=QMAX, fma=False):
    """ReLU, clamp, then rint(clip(fl(fl(v / s) + u), 0, qmax)), all in float32"""
    _, v = _v(x, mean, invstd, gamma, beta, fma)
    v = np.minimum(np.maximum(v, np.float32(0)), np.float32(act_max))
    t = (v / np.float32(q_scale)).astype(np.float32) + u.astype(np.float32)
    return np.rint(np.clip(t, np.float32(0), np.float32(qmax)))


def _slice_sums(a, splits):
    """[C, splits] sums over each slice's samples of a [B, C, HW] float64 array"""
    return np.stack([a[b0:b1].sum(axis=(0, 2)) for b0, b1 in slice_bounds(a.shape[0], splits)], axis=1)


def _ulps(got, ref):
    """|got - ref| in units of the float32 spacing at ref (ref float64)"""
    got = np.asarray(got, dtype=np.float64)
    return np.abs(got - ref) / np.spacing(np.abs(ref).astype(np.float32)).astype(np.float64)


def _records(scratch, C_):
    """the scratch as [C, ST_SPLITS, 2] partial sums and [C] counters"""
    rec = scratch[:scratch_bytes(C_)].cpu().numpy().view(np.float64).reshape(C_, ST_REC)
    return rec[:, :2 * ST_SPLITS].reshape(C_, ST_SPLITS, 2), rec[:, 2 * ST_SPLITS:].view(np.uint32)


# ---------------------------------------------------------------------------------------------- GPU plumbing

@pytest.fixture(scope="module")
def dev(lib):
    assert torch.cuda.is_available()
    yield torch.device("cuda:0")
    _profiled(lambda: None)     # one empty session last: the test files after this one start from a drained profiler


_KERNEL = re.compile(r"\b(k_pool_stats|k_chan_stats|k_bn_act_pack_tiled|k_bn_act_pack_lean|k_bn_act_pack|k_bn_bwd_stats|"
                     r"k_bn_bwd_apply_img|k_bn_bwd_apply_lean|k_bn_bwd_apply)\b(<[^>]*>)?")


def _profiled(fn):
    """fn() under torch.profiler -> (its result, the stage kernels recorded).  As in test_gpu_umma_sweep.py, the session
    first runs one marker kernel and waits 10 ms: the profiler was seen to start recording only after the first kernels of
    a session"""
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        torch.cuda._sleep(1000)
        torch.cuda.synchronize()
        time.sleep(0.01)
        out = fn()
        torch.cuda.synchronize()
    seen = set()
    for e in prof.events():
        m = _KERNEL.search(e.name) if e.device_type == torch.autograd.DeviceType.CUDA else None
        if m:
            seen.add(m.group(1) + (m.group(2) or ""))
    return out, seen


def _launch(expect, fn):
    """runs fn under torch.profiler: the stage kernels it launched must be exactly `expect`.  The dispatch is
    deterministic and every fn here recomputes the same outputs from the same inputs (running statistics restored
    first), so a session whose kernel set differs is profiled again, up to three times in all: a wrong dispatch fails
    every time."""
    for _ in range(3):
        out, seen = _profiled(fn)
        if seen == set(expect):
            break
    assert seen == set(expect), (sorted(seen), sorted(expect))
    return out


def _p(t):
    return None if t is None else t.data_ptr()


def _scratch(lib, dev, C_):
    return torch.zeros(int(lib.nn_stage_scratch_bytes(C_)) + 64, dtype=torch.uint8, device=dev)


def _fwd(lib, o, x, B, C_, H, W, pool, scratch, stats_ready=False, act=None, u=None, eval_mode=False):
    """nn_stage_fwd into the buffers of o (pooled, amax, gamma, beta, rm, rv, mean, invstd, xp, xmax)"""
    from noisynet_b200 import _lib
    a = _lib.StageArgs()
    a.in_ = x.data_ptr(); a.B, a.C, a.H, a.W, a.pool = B, C_, H, W, pool
    a.pooled, a.argmax = _p(o.get("pooled")), _p(o.get("amax"))
    a.gamma, a.beta, a.running_mean, a.running_var = _p(o["gamma"]), _p(o["beta"]), _p(o["rm"]), _p(o["rv"])
    a.momentum, a.eps = float(MOM), float(EPS)
    a.mean, a.invstd = _p(o["mean"]), _p(o["invstd"])
    a.act_max, a.q_bits, a.q_hi = ACT_MAX, BITS, Q_HI
    a.stochastic = 0.0 if eval_mode else STOCH
    a.u_inject = _p(u)
    a.rng = _lib.Rng(SEED, OFFSET, None)
    a.xp, a.Cp, a.act, a.xmax_out, a.scratch = _p(o["xp"]), o["xp"].shape[-1], _p(act), _p(o["xmax"]), _p(scratch)
    a.eval_mode, a.stats_ready = int(eval_mode), int(stats_ready)
    _lib.check(lib.nn_stage_fwd(C.byref(a), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_fwd")


def _bwd(lib, o, g, x, B, C_, H, W, pool, scratch, gyp, planes=None, gy_f32=None, act_max=ACT_MAX, q_hi=Q_HI):
    """nn_stage_bwd with the statistics and parameters of o (mean, invstd, gamma, beta) into o's dgamma / dbeta"""
    from noisynet_b200 import _lib
    b = _lib.StageBwdArgs()
    b.g, b.x, b.argmax = g.data_ptr(), x.data_ptr(), _p(o.get("amax"))
    b.B, b.C, b.H, b.W, b.pool = B, C_, H, W, pool
    b.mean, b.invstd, b.gamma, b.beta = _p(o["mean"]), _p(o["invstd"]), _p(o["gamma"]), _p(o["beta"])
    b.act_max, b.q_bits, b.q_hi = act_max, BITS, q_hi
    b.dgamma, b.dbeta = _p(o["dgamma"]), _p(o["dbeta"])
    b.gyp, b.Cp, b.gy_f32, b.scratch = gyp.data_ptr(), _pad8(C_), _p(gy_f32), _p(scratch)
    if planes is not None:
        b.gy_layout, b.virt_H, b.virt_W = _lib.PACK_SHIFT, planes[0], planes[1]
    _lib.check(lib.nn_stage_bwd(C.byref(b), 0, torch.cuda.current_stream().cuda_stream), "nn_stage_bwd")


def _pow2_gamma(C_, gen):
    return torch.tensor([-1.0, 0.5, 1.0, 2.0])[torch.randint(0, 4, (C_,), generator=gen)]


def _stage_buffers(dev, B, C_, PH, PW, gen):
    f = lambda *s: torch.empty(*s, device=dev)
    return dict(pooled=f(B, C_, PH, PW), amax=torch.empty(B, C_, PH, PW, dtype=torch.uint8, device=dev),
                gamma=_pow2_gamma(C_, gen).to(dev), beta=(torch.randn(C_, generator=gen) * 0.5).to(dev),
                rm=(torch.randn(C_, generator=gen) * 0.1).to(dev), rv=(torch.rand(C_, generator=gen) + 0.5).to(dev),
                mean=f(C_), invstd=f(C_), xp=torch.full((B, PH, PW, _pad8(C_)), 9.0, dtype=torch.bfloat16, device=dev),
                xmax=torch.full((1,), -1.0, device=dev), dgamma=f(C_), dbeta=f(C_))


# ---------------------------------------------------------------------------------------------- GPU tests: forward

def _check_codes(xp, want, C_, case):
    xp = xp.float().cpu().numpy()
    B = want.shape[0]
    got = xp.reshape(B, -1, xp.shape[-1])
    assert (got[..., C_:] == 0).all(), case                                   # padding channels
    bad = got[..., :C_].transpose(0, 2, 1) != want
    assert not bad.any(), "%s: %d codes differ, first at %s" % (case, int(bad.sum()), np.argwhere(bad)[0])


@pytest.mark.gpu
@pytest.mark.parametrize("case", FWD, ids=lambda c: "B%d-C%d-%dx%d-pool%d-ready%d" % c)
def test_stage_fwd(dev, lib, case):
    """pooling and argmax exactly; mean / invstd and the running statistics within 1 ulp of float64; the partial sums in
    the scratch exactly; the codes of the tiled / lean hot kernel and of the general kernel (Philox, injected draws,
    eval mode) bit for bit against the float32 restatement; padding channels zero; xmax exact"""
    B, C_, H, W, pool, ready = case
    gen = torch.Generator().manual_seed(sum(case))
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    HW, n = PH * PW, B * PH * PW
    x = (torch.randint(-16, 17, (B, C_, H, W), generator=gen).float() / 4.0).to(dev)
    o = _stage_buffers(dev, B, C_, PH, PW, gen)
    rm0, rv0 = o["rm"].clone(), o["rv"].clone()
    # ---- pooling: the first maximum of the window in row-major order wins
    xn = x.cpu().numpy()
    if pool:
        win = xn.reshape(B, C_, PH, 2, PW, 2).transpose(0, 1, 2, 4, 3, 5).reshape(B, C_, PH, PW, 4)
        bn_in, amax_ref = win.max(-1), win.argmax(-1)
        assert (win == bn_in[..., None]).sum(-1).max() > 1                    # tied windows present
    else:
        bn_in = xn
    bn_in = bn_in.reshape(B, C_, HW)
    s1 = bn_in.astype(np.float64)
    m_ref = s1.sum(axis=(0, 2)) / n
    var = np.maximum((s1 * s1).sum(axis=(0, 2)) / n - m_ref * m_ref, 0.0)
    inv_ref = 1.0 / np.sqrt(var + float(EPS))
    if ready:           # the conv launch produced the statistics (and zeroed xmax: run() does)
        o["mean"].copy_(torch.from_numpy(m_ref.astype(np.float32)))
        o["invstd"].copy_(torch.from_numpy(inv_ref.astype(np.float32)))
    scratch = _scratch(lib, dev, C_)

    def run(**kw):
        o["rm"].copy_(rm0); o["rv"].copy_(rv0)
        if ready:
            o["xmax"].zero_()
        _fwd(lib, o, x, B, C_, H, W, pool, scratch, stats_ready=ready, **kw)

    _launch(fwd_kernels(B, C_, H, W, pool, ready), run)
    if pool:
        assert np.array_equal(o["pooled"].cpu().numpy().reshape(B, C_, HW), bn_in)
        assert np.array_equal(o["amax"].cpu().numpy(), amax_ref)
    mean, invstd = o["mean"].cpu().numpy(), o["invstd"].cpu().numpy()
    if ready:
        assert torch.equal(o["rm"], rm0) and torch.equal(o["rv"], rv0)
    else:
        splits = stage_splits(n)
        assert _ulps(mean, m_ref).max() <= 1 and _ulps(invstd, inv_ref).max() <= 1
        mom = float(MOM)
        rm_ref = (1.0 - mom) * rm0.cpu().double().numpy() + mom * m_ref
        rv_ref = (1.0 - mom) * rv0.cpu().double().numpy() + mom * var * n / (n - 1)
        assert _ulps(o["rm"].cpu().numpy(), rm_ref).max() <= 1 and _ulps(o["rv"].cpu().numpy(), rv_ref).max() <= 1
        part, cnt = _records(scratch, C_)
        assert np.array_equal(part[:, :splits, 0], _slice_sums(s1, splits))
        assert np.array_equal(part[:, :splits, 1], _slice_sums(s1 * s1, splits))
        assert (part[:, splits:] == 0).all() and (cnt == 0).all()
    # ---- codes from the kernel's own statistics, Philox draws
    want = _codes(bn_in, mean, invstd, o["gamma"].cpu().numpy(), o["beta"].cpu().numpy(), _philox_u(B, C_, HW))
    _check_codes(o["xp"], want, C_, case)
    assert o["xmax"].item() == float(np.float32(want.max()) * Q_SCALE)
    hot = o["xp"].clone()
    stats = [o[k].clone() for k in ("mean", "invstd", "rm", "rv")]
    # ---- the general kernel (fp32 copy requested) on the same scratch: the same codes, statistics and copy
    o["xp"].fill_(9.0); o["xmax"].fill_(-1.0)
    act = torch.empty(B, C_, PH, PW, device=dev)
    _launch(fwd_kernels(B, C_, H, W, pool, ready, act=True), lambda: run(act=act))
    assert torch.equal(o["xp"], hot)
    assert all(torch.equal(o[k], t) for k, t in zip(("mean", "invstd", "rm", "rv"), stats))
    assert np.array_equal(act.cpu().numpy().reshape(B, C_, HW), (want * Q_SCALE).astype(np.float32))
    # ---- injected draws, anywhere in [-s, s)
    u = ((torch.rand(B, C_, PH, PW, generator=gen) * 2 - 1) * STOCH).to(dev)
    o["xp"].fill_(9.0); o["xmax"].fill_(-1.0)
    _launch(fwd_kernels(B, C_, H, W, pool, ready, u_inject=True), lambda: run(u=u))
    want_u = _codes(bn_in, mean, invstd, o["gamma"].cpu().numpy(), o["beta"].cpu().numpy(), u.cpu().numpy().reshape(B, C_, HW))
    _check_codes(o["xp"], want_u, C_, case)
    assert o["xmax"].item() == float(np.float32(want_u.max()) * Q_SCALE)
    if ready:
        return
    # ---- eval mode: the running statistics normalise, nothing updates, no rounding noise
    _launch(fwd_kernels(B, C_, H, W, pool, False, stoch=0.0), lambda: run(eval_mode=True))
    assert torch.equal(o["mean"], rm0) and torch.equal(o["rm"], rm0) and torch.equal(o["rv"], rv0)
    inv_eval = 1.0 / np.sqrt(rv0.cpu().double().numpy() + float(EPS))
    assert _ulps(o["invstd"].cpu().numpy(), inv_eval).max() <= 1
    want_e = _codes(bn_in, rm0.cpu().numpy(), o["invstd"].cpu().numpy(), o["gamma"].cpu().numpy(), o["beta"].cpu().numpy(),
                    np.zeros((1, 1, 1), np.float32))
    _check_codes(o["xp"], want_e, C_, case)


# ---------------------------------------------------------------------------------------------- GPU tests: backward

def _bwd_operands(B, C_, PH, PW, pool, gen):
    """v on a 1/4 grid over [-1, 6] (0, act_max and q_hi included), dyadic mean, power-of-two invstd and gamma: x, xhat
    and v are exact, and fl(fl(x - mean) * invstd) * gamma + beta gives v back"""
    k = torch.randint(-4, 25, (B, C_, PH, PW), generator=gen).double() / 4.0
    gamma = _pow2_gamma(C_, gen).double()
    beta = torch.randint(-8, 9, (C_,), generator=gen).double() / 8.0
    invstd = torch.tensor([0.5, 1.0, 2.0])[torch.randint(0, 3, (C_,), generator=gen)].double()
    mean = torch.randint(-16, 17, (C_,), generator=gen).double() / 8.0
    e = lambda t: t[None, :, None, None]
    x = (k - e(beta)) / e(gamma) / e(invstd) + e(mean)
    g = torch.randint(1, 9, (B, C_, PH, PW), generator=gen).float() * (torch.randint(0, 2, (B, C_, PH, PW), generator=gen) * 2 - 1)
    amax = torch.randint(0, 4, (B, C_, PH, PW), generator=gen, dtype=torch.uint8) if pool else None
    return x.float(), g, amax, mean.float(), invstd.float(), gamma.float(), beta.float()


def _bwd_reference(x, g, mean, invstd, gamma, beta, act_max, q_hi, fma=False):
    """the STE / clamp / ReLU masks (pass iff v > 0, v <= act_max, min(v, act_max) <= q_hi), and dv, xhat"""
    B, C_ = x.shape[:2]
    xhat, v = _v(x.reshape(B, C_, -1), mean, invstd, gamma, beta, fma)
    keep = (v > 0) & (v <= np.float32(act_max)) & (np.minimum(v, np.float32(act_max)) <= np.float32(q_hi))
    return np.where(keep, g.reshape(B, C_, -1), np.float32(0)), xhat, v


@pytest.mark.gpu
@pytest.mark.parametrize("case", BWD, ids=lambda c: "B%d-C%d-%dx%d-pool%d-planes%d" % c)
def test_stage_bwd(dev, lib, case):
    """masks exact at v = 0, act_max and q_hi (act_max below and above q_hi); dbeta / dgamma and the scratch partials exact
    (dyadic operands); gy_f32 within the rounding of k_bn_bwd_apply's fp32 formula; the packed gradient equal to
    bf16(gy_f32) at the argmax positions and zero at the others (planes: nothing written outside the outputs); the hot
    kernel bit-identical to the general one"""
    B, C_, H, W, pool, planes = case
    gen = torch.Generator().manual_seed(100 + sum(case))
    PH, PW = (H // 2, W // 2) if pool else (H, W)
    n, Cp = B * PH * PW, _pad8(C_)
    x, g, amax, mean, invstd, gamma, beta = _bwd_operands(B, C_, PH, PW, pool, gen)
    o = dict(mean=mean.to(dev), invstd=invstd.to(dev), gamma=gamma.to(dev), beta=beta.to(dev),
             amax=amax.to(dev) if pool else None, dgamma=torch.empty(C_, device=dev), dbeta=torch.empty(C_, device=dev))
    xd, gd = x.to(dev), g.to(dev)
    grid = PLANES_GRID[H] if planes else None
    splits = stage_splits(n)
    ic = np.float32(1.0) / (np.float32(B) * np.float32(PH) * np.float32(PW))
    for act_max in (3.0, ACT_MAX):                # act_max below q_hi: the clamp bound decides; above: the quantizer's
        dv, xhat, v = _bwd_reference(x.numpy(), g.numpy(), mean.numpy(), invstd.numpy(), gamma.numpy(), beta.numpy(), act_max, Q_HI)
        for edge in (0.0, act_max, Q_HI, act_max + 0.25, Q_HI + 0.25):
            assert (v == np.float32(edge)).sum() > 100
        outs = []
        for f32 in (False, True):
            scratch = _scratch(lib, dev, C_)
            if planes:
                plane_stride = (B * grid[0] * grid[1] + 127) // 128 * 128
                gyp = torch.full((Cp // 8, plane_stride, 8), 5.0, dtype=torch.bfloat16, device=dev)
            else:
                gyp = torch.full((B, H, W, Cp), 5.0, dtype=torch.bfloat16, device=dev)
            gyf = torch.full((B, C_, H, W), 5.0, device=dev) if f32 else None
            o["dgamma"].fill_(7.0); o["dbeta"].fill_(7.0)
            _launch(bwd_kernels(B, C_, H, W, pool, planes, f32),
                    lambda: _bwd(lib, o, gd, xd, B, C_, H, W, pool, scratch, gyp, planes=grid, gy_f32=gyf, act_max=act_max))
            outs.append((gyp, gyf, o["dgamma"].clone(), o["dbeta"].clone()))
            part, cnt = _records(scratch, C_)
            dv64, xh64 = dv.astype(np.float64), xhat.astype(np.float64)
            assert np.array_equal(part[:, :splits, 0], _slice_sums(dv64, splits))
            assert np.array_equal(part[:, :splits, 1], _slice_sums(dv64 * xh64, splits))
            assert (part[:, splits:] == 0).all() and (cnt == 0).all()
        (gyp, _, dg, db), (gyp_g, gyf, dg_g, db_g) = outs
        db_ref, dg_ref = dv64.sum(axis=(0, 2)), (dv64 * xh64).sum(axis=(0, 2))
        assert np.array_equal(db.cpu().numpy(), db_ref.astype(np.float32)) and np.array_equal(dg.cpu().numpy(), dg_ref.astype(np.float32))
        assert torch.equal(dg, dg_g) and torch.equal(db, db_g)
        assert torch.equal(gyp, gyp_g), "hot and general kernels differ"
        # gy_f32: d = gamma * invstd * (dv - dbeta * ic - xhat * dgamma * ic) in fp32.  gamma * invstd is a power of two
        # (exact); the bracket takes at most four roundings (two products, two differences; fewer with FMAs), each within
        # 2^-24 of a value no larger than |dv| + |dbeta ic| + |xhat dgamma ic|, so |d - D| <= 2^-22 |gamma invstd| (|dv| +
        # |dbeta ic| + |xhat dgamma ic|).  A wrong mask moves d by |gamma invstd g| >= |gamma invstd|, far outside it.
        e = lambda a: a.astype(np.float64)[None, :, None]
        a_ = e(db.cpu().numpy()) * float(ic)
        q_ = xh64 * e(dg.cpu().numpy()) * float(ic)
        gi = e(gamma.numpy()) * e(invstd.numpy())
        D = gi * (dv64 - a_ - q_)
        tol = 2.0 ** -22 * np.abs(gi) * (np.abs(dv64) + np.abs(a_) + np.abs(q_))
        gyf = gyf.cpu().numpy()
        if pool:
            am = amax.numpy().reshape(B, C_, PH, PW)
            full = np.zeros((B, C_, PH, 2, PW, 2), np.float64)
            sel = np.zeros((B, C_, PH, 2, PW, 2), bool)
            for q in range(4):
                sel[:, :, :, q >> 1, :, q & 1] = am == q
            full[sel] = np.broadcast_to(D.reshape(B, C_, PH, 1, PW, 1), full.shape)[sel]
            tolf = np.zeros_like(full)
            tolf[sel] = np.broadcast_to(tol.reshape(B, C_, PH, 1, PW, 1), full.shape)[sel]
            D_img, tol_img = full.reshape(B, C_, H, W), tolf.reshape(B, C_, H, W)
            assert (gyf.reshape(B, C_, PH, 2, PW, 2)[~sel] == 0).all()
        else:
            D_img, tol_img = D.reshape(B, C_, H, W), tol.reshape(B, C_, H, W)
        err = np.abs(gyf - D_img) - tol_img
        assert err.max() <= 0, "gy_f32 off by %.3e beyond the bound at %s" % (err.max(), np.unravel_index(err.argmax(), err.shape))
        # the packed gradient: bf16(gy_f32) at every output position (zeros at the non-argmax ones, zero padding channels)
        want = torch.zeros(B, Cp, H, W)
        want[:, :C_] = torch.from_numpy(gyf)
        want = want.to(torch.bfloat16)
        if planes:
            full_p = torch.full((Cp // 8, B, grid[0], grid[1], 8), 5.0, dtype=torch.bfloat16)
            full_p[:, :, :H, :W] = want.reshape(B, Cp // 8, 8, H, W).permute(1, 0, 3, 4, 2)
            got = gyp.cpu()
            assert torch.equal(got[:, :B * grid[0] * grid[1]].reshape(full_p.shape), full_p)
            assert bool((got[:, B * grid[0] * grid[1]:] == 5.0).all())
        else:
            assert torch.equal(gyp.cpu(), want.permute(0, 2, 3, 1))


# ---------------------------------------------------------------------------------------------- GPU tests: shared scratch

@pytest.mark.gpu
@pytest.mark.parametrize("B", [512, 768, 1024])
def test_shared_scratch_engine_sequence(dev, lib, B):
    """the engine's order on ONE scratch of nn_stage_scratch_bytes(390): forward bn1 (65 x 28 x 28 pooled), bn2 (120 x
    10 x 10 pooled), bn3 (390), backward bn3, bn2, bn1 (into conv1's planes), twice.  Every output must be bit-identical to
    the same calls on fresh scratches of their own.  bn2's statistics take 9 slices from batch 738 on and 12 at 1024:
    with the counters placed behind the calling stage's [C][16][2] partials they overwrote bn1's counters, and bn1's
    backward never wrote dgamma / dbeta."""
    gen = torch.Generator().manual_seed(B)
    stages = [("bn1", 65, 28, 1), ("bn2", 120, 10, 1), ("bn3", 390, 1, 0)]
    inputs = {}
    for name, C_, H, pool in stages:
        P = H // 2 if pool else H
        x = (torch.randn(B, C_, H, H, generator=gen) * 1.5 + 0.3).to(dev)
        gout = torch.randn(B, C_, P, P, generator=gen).to(dev)
        prm = (_pow2_gamma(C_, gen).to(dev), (torch.randn(C_, generator=gen) * 0.5).to(dev),
               (torch.randn(C_, generator=gen) * 0.1).to(dev), (torch.rand(C_, generator=gen) + 0.5).to(dev))
        inputs[name] = (x, gout, prm)
    worlds = {}
    for world in ("shared", "fresh"):
        st = {}
        for name, C_, H, pool in stages:
            P = H // 2 if pool else H
            o = _stage_buffers(dev, B, C_, P, P, gen)
            o["gamma"], o["beta"] = inputs[name][2][0], inputs[name][2][1]
            o["rm"], o["rv"] = inputs[name][2][2].clone(), inputs[name][2][3].clone()
            if name == "bn1":
                grid = PLANES_GRID[H]
                o["gyp"] = torch.zeros((_pad8(C_) // 8, (B * grid[0] * grid[1] + 127) // 128 * 128, 8), dtype=torch.bfloat16, device=dev)
            else:
                o["gyp"] = torch.empty(B, H, H, _pad8(C_), dtype=torch.bfloat16, device=dev)
            st[name] = o
        worlds[world] = st
    shared = _scratch(lib, dev, 390)
    for rep in range(2):
        for world, st in worlds.items():
            for o in st.values():
                for k in ("pooled", "mean", "invstd", "dgamma", "dbeta"):
                    o[k].fill_(-7.0)
                o["xp"].fill_(9.0); o["xmax"].fill_(-1.0)
                if o["gyp"].dim() == 4:
                    o["gyp"].fill_(3.0)
            sc = (lambda C_: shared) if world == "shared" else (lambda C_: _scratch(lib, dev, C_))
            for name, C_, H, pool in stages:
                _fwd(lib, st[name], inputs[name][0], B, C_, H, H, pool, sc(C_))
            for name, C_, H, pool in reversed(stages):
                o = st[name]
                _bwd(lib, o, inputs[name][1], o["pooled"] if pool else inputs[name][0], B, C_, H, H, pool, sc(C_), o["gyp"],
                     planes=PLANES_GRID[H] if name == "bn1" else None)
        torch.cuda.synchronize()
        bad = []
        for name, C_, H, pool in stages:
            a, b = worlds["shared"][name], worlds["fresh"][name]
            for k in ("pooled", "amax", "mean", "invstd", "rm", "rv", "xp", "xmax", "dgamma", "dbeta", "gyp"):
                if (pool or k not in ("pooled", "amax")) and not torch.equal(a[k], b[k]):
                    bad.append("%s.%s" % (name, k))
        assert not bad, "B=%d, pass %d: the shared scratch changed %s" % (B, rep, ", ".join(bad))
        assert bool((worlds["fresh"]["bn1"]["dgamma"] != -7.0).all())
