"""Every launch of NoisyNetEngine.train_step, as bench.py runs it, against float64 -- each launch recomputed from the
step's own input buffers for that launch.

One warm step, then one checked step per configuration (no injected draws: the fused bn3 epilogue and every Philox draw
are the benchmark's).  The engine's library handle is wrapped in a recorder that snapshots each call's argument
structs, so the test knows every launch's rng (seed, offset), scales, act_max, q_hi and pointers.  Everything the step
overwrites and a check needs (parameters, BatchNorm running statistics, AdamW moments, max|W|) is snapshotted before it.
Reading each launch's inputs from the step's own buffers keeps a discrete flip in one layer out of the next layer's
reference, so every bound below is derived from the launch's arithmetic, not from the spread of a whole step.  The
references run on the device in float64; Philox draws are restated by `_philox_t`, a torch port of
oracle.philox4x32_10 pinned against it on the CPU.  The step runs outside torch.profiler (a profiled multi-stream step
leaves later profiler sessions missing kernels); which kernel serves each launch is pinned by the sweeps.

  launch                                   check                                             bound
  nn_prepare_weights (2 launches)          wcodes of every layer vs float32 restatement      exact (Philox u of the layer's rng)
  nn_input_quant_pack_rows                 xp1 and the row-plane image                       exact (Philox u)
  nn_noisy_conv_fwd conv1 (pool + bn1)     pool1 vs max-pool of main + sigma z               NOISE_TOL
                                           amax1 where the window's top-two gap > 2 NOISE_TOL exact
                                           bn1 mean / invstd / running stats vs float64      L 2^-24 sum|x| (fp32 per-CTA chains)
  nn_stage_fwd bn1 / bn2 / bn3             xp2 / xp3 / xp4 vs float32 restatement            exact (either FMA contraction)
                                           pool2 / amax2 vs max-pool of y2n                  exact
                                           bn2 statistics vs float64 of pool2                1 ulp
                                           xmax2 / xmax4                                     exact
  nn_noisy_conv_fwd conv2 / fc1 / fc2      y2n / l1n / l2n vs main + sigma z                 NOISE_TOL (+ FP32_SUM on bf16 operands)
                                           bn3 statistics from fc1's split-K epilogue        umma sweep's _check_bn
                                           (unfused, B > 512: from the stage, vs float64)    1 ulp
  nn_head_fwd_bwd                          loss, g4, dgamma, dbeta; bn4 running stats        2^-17 of the terms; 1 ulp
                                           gyp4                                              == bf16(g4)
  nn_noisy_conv_wgrad x 4                  W.grad vs float64 of the packed operands, STE     FP32_SUM
  nn_noisy_conv_dgrad x 2, _dgrad_planes   gx4 / gx3 / gx2 vs float64 of the packed operands FP32_SUM
  nn_stage_bwd bn3 / bn2 / bn1             gyp3 / gyp2 / gyp1 (planes) vs stage sweep bound  bf16 of [D - tol, D + tol]
                                           pool routing, planes outside 28 x 28              exact zeros
                                           dgamma / dbeta                                    2^-22 sum |terms|
  step_part x 2 (AdamW, side + main)       every parameter and exp_avg vs float64 AdamW      2^-21 (|w| + |update|), 2^-22
                                           opt.absmax                                        == max|W| exactly

NOISE_TOL = main + 2^-22 |ref| + sigma (2e-3 + |z| (K/2 + 8) 2^-24): the fp32 rounding of the output, the MUFU
Box-Muller error bound of test_philox_normal_epilogue_matches_spec (2e-3 absolute on z), and the fp32 sum of the K sigma
products.  FP32_SUM = n 2^-24 sum |a b| * scale: the standard bound of an fp32 accumulation of n products.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from test_gpu_stage_sweep import _bwd_reference, _codes, _philox_u, _v
from test_gpu_umma_sweep import _check_bn

U24 = 2.0 ** -24
MUFU_Z = 2e-3                    # |z - z_spec| of the MUFU Box-Muller (test_philox_normal_epilogue_matches_spec)
DISTINCT = dict(act_max=(5.0, 4.0, 6.0), q_hi2=3.5, q_hi4=4.5, currents=[1.0, 2.0, 0.5, 3.0])
CONFIGS = {"q4-512": ("q4", 512, False), "q4-1024": ("q4", 1024, False), "q4-2048": ("q4", 2048, False),
           "distinct-768": ("q4", 768, True), "fp-512": ("fp", 512, False)}
EXPECTED_CALLS = {"nn_prepare_weights": 2, "nn_input_quant_pack_rows": 1, "nn_noisy_conv_fwd": 4, "nn_stage_fwd": 3,
                  "nn_head_fwd_bwd": 1, "nn_noisy_conv_wgrad": 4, "nn_noisy_conv_dgrad": 2, "nn_conv_dgrad_planes": 1,
                  "nn_stage_bwd": 3, "step_part": 2}


# ---------------------------------------------------------------------------------------------- Philox on the device

_M0, _M1, _W0, _W1, _MASK = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85, 0xFFFFFFFF


def _mulhilo(a, m):
    """(hi, lo) 32-bit words of a * m for int64 tensors a < 2^32 and a constant m < 2^32, without int64 overflow"""
    t1, t2 = (a & 0xFFFF) * m, (a >> 16) * m                 # both < 2^48
    s = t1 + ((t2 & 0xFFFF) << 16)
    return (t2 >> 16) + (s >> 32), s & _MASK


def _philox_t(group, seed, offset):
    """oracle.philox4x32_10 on int64 torch tensors: group -> [..., 4] words in [0, 2^32)"""
    c0 = torch.full_like(group, offset & _MASK)
    c1 = torch.full_like(group, (offset >> 32) & _MASK)
    c2, c3 = group & _MASK, (group >> 32) & _MASK
    k0, k1 = seed & _MASK, (seed >> 32) & _MASK
    for _ in range(10):
        hi0, lo0 = _mulhilo(c0, _M0)
        hi1, lo1 = _mulhilo(c2, _M1)
        c0, c1, c2, c3 = (hi1 ^ c1 ^ k0) & _MASK, lo1, (hi0 ^ c3 ^ k1) & _MASK, lo0
        k0, k1 = (k0 + _W0) & _MASK, (k1 + _W1) & _MASK
    return torch.stack([c0, c1, c2, c3], dim=-1)


def _u01_t(r):
    return (r >> 8).to(torch.float32) * (2.0 ** -24)


def _usym_t(r, s):
    """nn_usym: fl(fl(u01 * fl(2s)) - s)"""
    s32 = torch.tensor(s, dtype=torch.float32, device=r.device)
    return _u01_t(r) * (2.0 * s32) - s32


def _normal_mn_t(M, N, seed, offset, dev):
    """oracle.philox_normal_mn on the device (exact transcendentals in float64): [M, N] float64"""
    ng = (N + 3) // 4
    g = torch.arange(M, dtype=torch.int64, device=dev)[:, None] * ng + torch.arange(ng, dtype=torch.int64, device=dev)[None, :]
    r = _philox_t(g, seed, offset)
    out = torch.empty(r.shape, dtype=torch.float64, device=dev)
    two_pi, m_pi = float(np.float32(6.2831853071795865)), float(np.float32(-3.14159265358979324))
    for j in (0, 2):
        u1 = (r[..., j].to(torch.float32).double() * 2.0 ** -32 + 2.0 ** -33).float().double()
        u2 = _u01_t(r[..., j + 1]).double()
        rad = torch.sqrt(-2.0 * torch.log(u1))
        th = (u2 * two_pi + m_pi).float().double()
        out[..., j] = (rad * torch.cos(th)).float().double()
        out[..., j + 1] = (rad * torch.sin(th)).float().double()
    return out.reshape(M, ng * 4)[:, :N]


# ---------------------------------------------------------------------------------------------- restatements

def weight_codes(w, q_bits, q_hi, stoch, seed, offset):
    """k_quant_codes: codes 2k - qmax, k = rint(clip(fl(fl(fl(w + q_hi) / s) + u), 0, qmax)), s = fl32(2 q_hi / qmax),
    u of element idx = usym(Philox group idx / 4, word idx % 4)"""
    qmax = float(2 ** q_bits - 1)
    s = torch.tensor(max(2.0 * q_hi / qmax, 1e-6), dtype=torch.float32, device=w.device)
    flat = w.reshape(-1).float()
    n = flat.numel()
    u = _usym_t(_philox_t(torch.arange((n + 3) // 4, dtype=torch.int64, device=w.device), seed, offset), stoch).reshape(-1)[:n]
    t = (flat + torch.tensor(q_hi, dtype=torch.float32, device=w.device)) / s + u
    k = torch.round(t.clamp(0.0, qmax))
    return (2.0 * k - qmax).to(torch.int8)


def input_codes(x, q_bits, q_hi, stoch, seed, offset):
    """k_quant_pack_input / the rows kernel: the codes [B, C, H, W] of x; pixel p (NCHW b, h, w) draws group 2p + c / 4,
    word c % 4 (one chunk of 8 channels)"""
    B, Cc, H, W = x.shape
    qmax = float(2 ** q_bits - 1)
    s = torch.tensor(max(q_hi / qmax, 1e-6), dtype=torch.float32, device=x.device)
    pix = torch.arange(B * H * W, dtype=torch.int64, device=x.device)
    r = _philox_t(torch.stack([2 * pix, 2 * pix + 1], dim=-1), seed, offset).reshape(B * H * W, 8)[:, :Cc]
    u = _usym_t(r, stoch).reshape(B, H, W, Cc).permute(0, 3, 1, 2)
    return torch.round((x.float() / s + u).clamp(0.0, qmax))


def _rows_ref(codes, kw, n_planes):
    """the row-plane image [P, B, H, W, 8] of codes [B, C, H, W] (test_gpu_shift_rows.rows_ref, on the device)"""
    B, Cc, H, W = codes.shape
    out = torch.zeros(n_planes * 8, B, H, W, dtype=codes.dtype, device=codes.device)
    for e in range(min(n_planes * 8, kw * Cc)):
        k, c = divmod(e, Cc)
        out[e, :, :, :W - k] = codes[:, c, :, k:]
    return out.reshape(n_planes, 8, B, H, W).permute(0, 2, 3, 4, 1)


class Report:
    """per-check worst error / bound ratios; a ratio > 1 fails"""

    def __init__(self):
        self.rows, self.bad = [], []

    def within(self, name, got, ref, tol, mask=None):
        d = (got.double() - ref).abs()
        if mask is not None:
            d, tol = d[mask], tol[mask]
        ratio = d / tol.clamp_min(1e-300)
        worst = float(ratio.max()) if ratio.numel() else 0.0
        i = int(ratio.argmax()) if ratio.numel() else 0
        self.rows.append((name, float(d.max()) if d.numel() else 0.0, float(tol.reshape(-1)[i]) if tol.numel() else 0.0, worst))
        if worst > 1.0:
            self.bad.append("%s: %d values beyond the bound, worst %.3e vs %.3e" % (
                name, int((ratio > 1).sum()), float(d.reshape(-1)[i]), float(tol.reshape(-1)[i])))

    def exact(self, name, got, want, mask=None):
        eq = got == want
        if mask is not None:
            eq = eq | ~mask
        n = int((~eq).sum())
        self.rows.append((name, float(n), 0.0, float(n)))
        if n:
            self.bad.append("%s: %d values differ, first at %s" % (name, n, tuple(int(v) for v in torch.nonzero(~eq)[0])))

    def true(self, name, cond, what=""):
        self.rows.append((name, 0.0 if cond else 1.0, 0.0, 0.0 if cond else 1.0))
        if not cond:
            self.bad.append("%s: %s" % (name, what))


# ---------------------------------------------------------------------------------------------- the step

class _Recorder:
    """the engine's library handle: records every call with a snapshot of its argument structs"""

    def __init__(self, lib):
        self._lib, self.calls = lib, []

    def __getattr__(self, name):
        fn = getattr(self._lib, name)

        def call(*args):
            self.calls.append((name, [_snap(name, a, args) for a in args]))
            return fn(*args)
        return call


def _snap(name, a, args):
    from noisynet_b200._lib import WPrepJob
    obj = a._obj if type(a).__name__ == "CArgObject" else a
    if name == "nn_prepare_weights" and a is args[0]:
        n = int(args[1])
        return (WPrepJob * n).from_buffer_copy(C.string_at(C.addressof(obj), n * C.sizeof(WPrepJob)))
    if isinstance(obj, (C.Structure, C.Array)):
        return type(obj).from_buffer_copy(obj)
    return obj


def _expected(cfg):
    variant, B, distinct = cfg
    q = 4 if variant == "q4" else 0
    am = DISTINCT["act_max"] if distinct else (5.0, 5.0, 5.0)
    qh = (1.0, DISTINCT["q_hi2"] if distinct else 5.0, 5.0, DISTINCT["q_hi4"] if distinct else 5.0) if q else (0.0,) * 4
    cur = DISTINCT["currents"] if distinct else [1.0] * 4
    a_cs = [float(np.float32(max(h / 15.0, 1e-6))) if q else 0.0 for h in qh]
    w_cs = float(np.float32(2.0 / 15.0)) / 2.0 if q else 0.0
    return dict(q=q, B=B, act_max=am, q_hi=qh, currents=cur, a_cs=a_cs, w_cs=w_cs)


def run_step(dev, cid):
    """builds bench.py's model for configuration cid, runs a warm step and one recorded step -> state dict"""
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, init_like_reference, make_fused_optimizer, with_quant
    cfg = CONFIGS[cid]
    E = _expected(cfg)
    B = E["B"]
    torch.manual_seed(1000 + B + (7 if cfg[2] else 0))
    a = default_args()
    if E["q"]:
        with_quant(a, 4, 4)
    if cfg[2]:
        a.act_max1, a.act_max2, a.act_max3 = DISTINCT["act_max"]
        a.layer_currents = list(DISTINCT["currents"])
    m = init_like_reference(NoisyNet(a, fused=True, precision="bf16")).to(dev)
    if E["q"]:
        m.quantize2.running_max = torch.tensor(E["q_hi"][1], device=dev)
        m.quantize4.running_max = torch.tensor(E["q_hi"][3], device=dev)
    m.collect_stats = False
    m.train()
    opt = make_fused_optimizer(m, a)
    eng = NoisyNetEngine(m, B, opt=opt)
    gen = torch.Generator().manual_seed(B)
    xs = [(torch.randint(0, 16, (B, 3, 32, 32), generator=gen).float() / 15).to(dev) for _ in range(2)]
    ys = [torch.randint(0, 10, (B,), generator=gen).to(dev) for _ in range(2)]
    eng.train_step(xs[0], ys[0])
    torch.cuda.synchronize()
    names = [n for n, _ in m.named_parameters()]
    params = dict(m.named_parameters())
    S = dict(cid=cid, E=E, eng=eng, m=m, opt=opt, x=xs[1], labels=ys[1])
    S["pre"] = {n: p.detach().clone() for n, p in params.items()}
    S["pre_m"] = {n: opt.state[p]["exp_avg"].clone() for n, p in params.items()}
    S["pre_v"] = {n: opt.state[p]["exp_avg_sq"].clone() for n, p in params.items()}
    S["pre_step"] = int(opt.step_dev.item())
    S["pre_absmax"] = opt.absmax.clone()
    S["pre_bn"] = {k: (getattr(m, k).running_mean.clone(), getattr(m, k).running_var.clone()) for k in ("bn1", "bn2", "bn3", "bn4")}
    rec = _Recorder(eng.lib)
    part = opt.step_part

    def step_part(ps, advance):
        rec.calls.append(("step_part", [[names[[id(q) for q in params.values()].index(id(p))] for p in ps], advance]))
        return part(ps, advance)
    eng.lib, opt.step_part = rec, step_part
    try:
        eng.train_step(xs[1], ys[1])
        torch.cuda.synchronize()
    finally:
        eng.lib = rec._lib
        del opt.step_part
    assert ops.error_flag() == 0
    S["calls"] = rec.calls
    S["fuse_bn3"] = eng.fuse_bn3
    # the outputs the checks read, copied: the sensitivity test perturbs copies of this dict
    for k in ("xp1", "x1_planes", "pool1", "amax1", "xp2", "xmax2", "y2n", "pool2", "amax2", "xp3", "l1n", "xp4", "xmax4", "l2n",
              "loss", "g4", "gyp4", "gx4", "gyp3", "gx3", "gyp2", "gx2", "gyp1"):
        S[k] = getattr(eng, k).clone()
    S["stat"] = {k: (v[0].clone(), v[1].clone()) for k, v in eng.stat.items()}
    S["wcodes"] = {k: v.clone() for k, v in eng.wcodes.items()}
    S["post"] = {n: p.detach().clone() for n, p in params.items()}
    S["grad"] = {n: p.grad.clone() for n, p in params.items()}
    S["post_m"] = {n: opt.state[p]["exp_avg"].clone() for n, p in params.items()}
    S["absmax"] = opt.absmax.clone()
    S["bn"] = {k: (getattr(m, k).running_mean.clone(), getattr(m, k).running_var.clone()) for k in ("bn1", "bn2", "bn3", "bn4")}
    return S


def _calls(S, name):
    return [args for n, args in S["calls"] if n == name]


WEIGHTS = ("conv1.weight", "conv2.weight", "linear1.weight", "linear2.weight")


# ---------------------------------------------------------------------------------------------- checks

def check_coverage(S, R):
    got = {}
    for n, _ in S["calls"]:
        got[n] = got.get(n, 0) + 1
    R.true("coverage", got == EXPECTED_CALLS, "entry points %s, checked %s" % (sorted(got.items()), sorted(EXPECTED_CALLS.items())))


def check_weight_codes(S, R):
    E = S["E"]
    jobs = [j for args in _calls(S, "nn_prepare_weights") for j in args[0]]
    R.true("prepare.jobs", len(jobs) == 7, "%d jobs" % len(jobs))
    if not E["q"]:
        return
    for li, name in enumerate(WEIGHTS):
        w = S["pre"][name]
        mine = [j for j in jobs if j.w_raw == S["m"].get_parameter(name).data_ptr()]
        R.true("prepare.%s.jobs" % name, len(mine) == (1 if li == 0 else 2) and all(
            j.q_bits == E["q"] and j.q_hi == 1.0 and j.stochastic == 0.5 and j.codes == S["eng"].wcodes[li].data_ptr()
            and (j.rng.seed, j.rng.offset) == (mine[0].rng.seed, mine[0].rng.offset) for j in mine), "job arguments")
        want = weight_codes(w, E["q"], 1.0, 0.5, mine[0].rng.seed, mine[0].rng.offset)
        R.exact("prepare.%s.codes" % name, S["wcodes"][li][:w.numel()], want)


def check_input_pack(S, R):
    E, eng = S["E"], S["eng"]
    (args,) = _calls(S, "nn_input_quant_pack_rows")
    rng = args[12]
    R.true("input.args", args[0] == S["x"].data_ptr() and args[1] == eng.xp1.data_ptr() and args[2] == eng.x1_planes.data_ptr()
           and args[8] == E["q"] and args[9] == E["q_hi"][0] and (args[10] == 0.5 if E["q"] else True), "arguments")
    B = E["B"]
    if E["q"]:
        codes = input_codes(S["x"], E["q"], 1.0, 0.5, rng.seed, rng.offset)
    else:
        codes = S["x"].to(torch.bfloat16).float()
    xp = S["xp1"].float()
    R.exact("input.xp1", xp[..., :3].permute(0, 3, 1, 2), codes)
    R.exact("input.xp1.pad", xp[..., 3:], torch.zeros_like(xp[..., 3:]))
    n_planes = 2
    pl = S["x1_planes"][:n_planes * B * 32 * 32 * 8].reshape(n_planes, B, 32, 32, 8).float()
    R.exact("input.planes", pl, _rows_ref(codes, 5, n_planes))


def _x_values(S, key, C_):
    """the forward operand of a GEMM: NHWC bf16 codes (or bf16 values) -> NCHW float64"""
    xp = S[key]
    if xp.dim() == 2:
        return xp[:, :C_].double()[:, :, None, None]
    return xp[..., :C_].permute(0, 3, 1, 2).double()


def _w_main(S, li):
    """the weight operand: int8 codes 2k - qmax (q > 0) or bf16(W), [Cout, Cin, KH, KW] float64"""
    w = S["pre"][WEIGHTS[li]]
    shape = {0: (65, 3, 5, 5), 1: (120, 65, 5, 5), 2: (390, 120, 5, 5), 3: (10, 390, 1, 1)}[li]
    if S["E"]["q"]:
        return S["wcodes"][li][:w.numel()].double().reshape(shape)
    return w.to(torch.bfloat16).double().reshape(shape)


def _noisy_ref(S, li, x, scale_val, mode_merged, fwd):
    """main + sigma z and NOISE_TOL for layer li: x [B, Cin, H, W] codes / values (float64), the output [B, Cout, OH, OW]"""
    E = S["E"]
    a_cs, w_cs = E["a_cs"][li] or 1.0, E["w_cs"] or 1.0
    wm = _w_main(S, li)
    K = wm[0].numel()
    main = F.conv2d(x, wm) * (a_cs * w_cs)
    tol = 2.0 ** -23 * main.abs()
    if not E["q"]:
        tol = tol + K * U24 * F.conv2d(x.abs(), wm.abs())
    a = S["pre"][WEIGHTS[li]].abs().reshape(wm.shape).float()
    g = (a if mode_merged else a * a + a).to(torch.bfloat16).double()
    Ssum = F.conv2d(x * (E["a_cs"][li] or 1.0), g)
    coef = float(np.float32(0.1) * (np.float32(scale_val) / np.float32(E["currents"][li])))
    sigma = torch.sqrt(coef * Ssum)
    B, N, OH, OW = main.shape
    z = _normal_mn_t(B * OH * OW, N, fwd.rng.seed, fwd.rng.offset, x.device).reshape(B, OH, OW, N).permute(0, 3, 1, 2)
    ref = main + z * sigma
    tol = tol + 2.0 ** -22 * ref.abs() + sigma * (MUFU_Z + z.abs() * (K / 2 + 8) * U24) + 1e-30
    return ref, tol


def _fwd_args(S):
    return [args[0] for args in _calls(S, "nn_noisy_conv_fwd")]


def _fwd_wiring(S, R, li, fwd, x_ptr, a_cs):
    E = S["E"]
    R.true("fwd%d.args" % li, fwd.x_packed == x_ptr and fwd.a_code_scale == np.float32(a_cs) and fwd.w_code_scale == np.float32(E["w_cs"])
           and fwd.current == np.float32(E["currents"][li]) and fwd.z_inject is None, "arguments")


def check_conv1(S, R):
    E, eng = S["E"], S["eng"]
    fwd = _fwd_args(S)[0]
    _fwd_wiring(S, R, 0, fwd, eng.x1_planes.data_ptr(), E["a_cs"][0])
    R.true("conv1.out", fwd.pooled_out == eng.pool1.data_ptr() and fwd.argmax_out == eng.amax1.data_ptr()
           and fwd.bn_mean == eng.stat["bn1"][0].data_ptr() and fwd.zero_out == eng.xmax2.data_ptr(), "output pointers")
    x = _x_values(S, "xp1", 3)
    ref, tol = _noisy_ref(S, 0, x, float(S["pre_absmax"][0]), True, fwd)
    B = E["B"]
    win = ref.reshape(B, 65, 14, 2, 14, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, 65, 14, 14, 4)
    twin = tol.reshape(B, 65, 14, 2, 14, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, 65, 14, 14, 4).amax(-1)
    pv, pi = win.max(-1)
    R.within("conv1.pool1", S["pool1"], pv, twin)
    top2 = win.topk(2, dim=-1).values
    clear = (top2[..., 0] - top2[..., 1]) > 2 * twin
    R.true("conv1.amax1.clear", float(clear.double().mean()) > 0.9, "too few clear windows")
    R.exact("conv1.amax1", S["amax1"].long(), pi, mask=clear)
    # bn1 statistics against float64 of the step's own pool1.  The kernel sums each channel in fp32 per thread over the
    # tiles of its CTA (block tiles of 16 x 8 outputs: 32 pooled values per channel, 8 tiles per 28 x 28 image), then
    # in float64 over CTAs; an fp32 chain of L terms errs by at most L 2^-24 sum|x|.  L = 32 ceil(8 B / SMs), doubled for
    # an uneven deal of tiles.
    p = S["pool1"].double()
    n = B * 196
    sms = torch.cuda.get_device_properties(p.device).multi_processor_count
    L = 2 * 32 * math.ceil(8 * B / sms)
    m_ref = p.sum((0, 2, 3)) / n
    e2 = (p * p).sum((0, 2, 3)) / n
    var = (e2 - m_ref * m_ref).clamp_min(0)
    t1 = L * U24 * p.abs().sum((0, 2, 3)) / n
    t2 = L * U24 * e2
    tv = t2 + 2 * m_ref.abs() * t1 + t1 * t1
    inv = 1.0 / torch.sqrt(var + float(np.float32(1e-5)))
    mean, invstd = S["stat"]["bn1"]
    R.within("bn1.mean", mean, m_ref, t1 + U24 * m_ref.abs())
    R.within("bn1.invstd", invstd, inv, 0.5 * inv ** 3 * tv + 2 * U24 * inv)
    mom = float(np.float32(0.1))
    rm0, rv0 = S["pre_bn"]["bn1"]
    rm, rv = S["bn"]["bn1"]
    R.within("bn1.running_mean", rm, (1 - mom) * rm0.double() + mom * m_ref, mom * t1 + 2 * U24 * rm.double().abs() + 1e-30)
    R.within("bn1.running_var", rv, (1 - mom) * rv0.double() + mom * var * n / (n - 1), mom * tv * n / (n - 1) + 2 * U24 * rv.double().abs())


def _stage_codes(S, R, name, inp, C_, HW, mean, invstd, key_bn, act_max, q_hi, sf, out_key):
    """codes of one stage forward from the step's own input and statistics, against either FMA contraction"""
    E, B = S["E"], S["E"]["B"]
    gamma = S["pre"][key_bn + ".weight"].cpu().numpy()
    beta = S["pre"][key_bn + ".bias"].cpu().numpy()
    x = inp.reshape(B, C_, HW).cpu().numpy()
    mn, iv = mean.cpu().numpy(), invstd.cpu().numpy()
    xp = S[out_key].float().cpu().numpy().reshape(B, HW, -1)
    got = xp[..., :C_].transpose(0, 2, 1)
    if E["q"]:
        qs = np.float32(q_hi / 15.0)
        u = _philox_u(B, C_, HW, sf.rng.seed, sf.rng.offset, 0.5)
        wants = [_codes(x, mn, iv, gamma, beta, u, act_max, qs, np.float32(15), fma=f) for f in (False, True)]
        vals = [w * qs for w in wants]
    else:
        vals = [np.minimum(np.maximum(_v(x, mn, iv, gamma, beta, f)[1], np.float32(0)), np.float32(act_max)) for f in (False, True)]
        wants = [torch.from_numpy(v).to(torch.bfloat16).float().numpy() for v in vals]
    ok = (got == wants[0]) | (got == wants[1])
    R.exact(name + ".codes", torch.from_numpy(ok), torch.ones_like(torch.from_numpy(ok)))
    R.exact(name + ".pad", torch.from_numpy(xp[..., C_:]), torch.zeros(xp[..., C_:].shape))
    return vals, got


def _stage_wiring(S, R, name, sf, in_ptr, xp_ptr, act_max, q_hi, key):
    E, eng = S["E"], S["eng"]
    R.true(name + ".args", sf.in_ == in_ptr and sf.xp == xp_ptr and sf.act_max == np.float32(act_max) and sf.q_hi == q_hi
           and sf.q_bits == E["q"] and sf.mean == eng.stat[key][0].data_ptr() and sf.u_inject is None
           and (sf.stochastic == 0.5 if E["q"] else True), "arguments")


def check_stage_fwd(S, R):
    E, eng, B = S["E"], S["eng"], S["E"]["B"]
    am, qh = E["act_max"], E["q_hi"]
    sf = [args[0] for args in _calls(S, "nn_stage_fwd")]
    # bn1 (statistics from conv1)
    _stage_wiring(S, R, "stage1", sf[0], eng.pool1.data_ptr(), eng.xp2.data_ptr(), am[0], qh[1], "bn1")
    R.true("stage1.ready", sf[0].stats_ready == 1 and sf[0].xmax_out == eng.xmax2.data_ptr(), "stats_ready / xmax")
    vals, got = _stage_codes(S, R, "stage1", S["pool1"], 65, 196, *S["stat"]["bn1"], "bn1", am[0], qh[1], sf[0], "xp2")
    xm = [float(np.float32(v.max())) for v in vals]
    R.true("stage1.xmax2", float(S["xmax2"]) in xm, "%r not in %r" % (float(S["xmax2"]), xm))
    # bn2: pooling of y2n, statistics of pool2
    _stage_wiring(S, R, "stage2", sf[1], eng.y2n.data_ptr(), eng.xp3.data_ptr(), am[1], qh[2], "bn2")
    y = S["y2n"]
    win = y.reshape(B, 120, 5, 2, 5, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, 120, 5, 5, 4)
    pv, pi = win.max(-1)
    R.exact("stage2.pool2", S["pool2"], pv)
    R.exact("stage2.amax2", S["amax2"].long(), pi)
    _stage_stats(S, R, "bn2", S["pool2"])
    _stage_codes(S, R, "stage2", S["pool2"], 120, 25, *S["stat"]["bn2"], "bn2", am[1], qh[2], sf[1], "xp3")
    # bn3: statistics from fc1's split-K epilogue where the library fuses them (M = B <= 512 for 390 channels on an
    # H100), from the stage itself otherwise
    _stage_wiring(S, R, "stage3", sf[2], eng.l1n.data_ptr(), eng.xp4.data_ptr(), am[2], qh[3], "bn3")
    R.true("stage3.ready", sf[2].stats_ready == int(S["fuse_bn3"]) and sf[2].xmax_out == eng.xmax4.data_ptr(), "stats_ready / xmax")
    if not S["fuse_bn3"]:
        _stage_stats(S, R, "bn3", S["l1n"][:, :, None, None])
    vals, _ = _stage_codes(S, R, "stage3", S["l1n"], 390, 1, *S["stat"]["bn3"], "bn3", am[2], qh[3], sf[2], "xp4")
    xm = [float(np.float32(v.max())) for v in vals]
    R.true("stage3.xmax4", float(S["xmax4"]) in xm, "%r not in %r" % (float(S["xmax4"]), xm))


def _stage_stats(S, R, key, p):
    """statistics the stage kernel computes itself (float64 sums of fp32 values): within 1 ulp of float64"""
    p = p.double()
    n = p.shape[0] * p.shape[2] * p.shape[3]
    m_ref = p.sum((0, 2, 3)) / n
    var = ((p * p).sum((0, 2, 3)) / n - m_ref * m_ref).clamp_min(0)
    inv = 1.0 / torch.sqrt(var + float(np.float32(1e-5)))
    mean, invstd = S["stat"][key]
    R.within(key + ".mean", mean, m_ref, _ulp(m_ref))
    R.within(key + ".invstd", invstd, inv, _ulp(inv))
    mom = float(np.float32(0.1))
    rm0, rv0 = S["pre_bn"][key]
    rm, rv = S["bn"][key]
    rmr, rvr = (1 - mom) * rm0.double() + mom * m_ref, (1 - mom) * rv0.double() + mom * var * n / (n - 1)
    R.within(key + ".running_mean", rm, rmr, _ulp(rmr))
    R.within(key + ".running_var", rv, rvr, _ulp(rvr))


def _ulp(ref):
    return torch.from_numpy(np.spacing(np.abs(ref.cpu().numpy()).astype(np.float32)).astype(np.float64)).to(ref.device)


def check_fwd_gemms(S, R):
    E, eng, B = S["E"], S["eng"], S["E"]["B"]
    fwd = _fwd_args(S)
    # conv2: x = stage 1's codes, external DAC, scale = xmax2
    _fwd_wiring(S, R, 1, fwd[1], eng.xp2.data_ptr(), E["a_cs"][1])
    R.true("conv2.scale", fwd[1].scale_dev == eng.xmax2.data_ptr() and fwd[1].y_noisy == eng.y2n.data_ptr(), "scale / output")
    ref, tol = _noisy_ref(S, 1, _x_values(S, "xp2", 65), float(S["xmax2"]), False, fwd[1])
    R.within("conv2.y2n", S["y2n"], ref, tol)
    # fc1: a 5 x 5 conv over the NHWC pooled codes, merged DAC, scale = max|W3|, bn3 statistics in the split-K epilogue
    _fwd_wiring(S, R, 2, fwd[2], eng.xp3.data_ptr(), E["a_cs"][2])
    fused = S["fuse_bn3"]
    R.true("fc1.bn", (fwd[2].bn_mean, fwd[2].zero_out) == ((eng.stat["bn3"][0].data_ptr(), eng.xmax4.data_ptr()) if fused else (None, None)),
           "fused bn3")
    ref, tol = _noisy_ref(S, 2, _x_values(S, "xp3", 120), float(S["pre_absmax"][2]), True, fwd[2])
    R.within("fc1.l1n", S["l1n"], ref.reshape(B, 390), tol.reshape(B, 390))
    if fused:
        try:
            _check_bn(S["l1n"], *S["stat"]["bn3"])
            R.true("bn3.stats", True)
        except AssertionError:
            R.true("bn3.stats", False, "mean / invstd beyond _check_bn's bound")
    # fc2: external DAC, scale = xmax4
    _fwd_wiring(S, R, 3, fwd[3], eng.xp4.data_ptr(), E["a_cs"][3])
    ref, tol = _noisy_ref(S, 3, _x_values(S, "xp4", 390), float(S["xmax4"]), False, fwd[3])
    R.within("fc2.l2n", S["l2n"], ref.reshape(B, 10), tol.reshape(B, 10))


def check_head(S, R):
    B = S["E"]["B"]
    z = S["l2n"].double()
    lab = S["labels"]
    m = z.mean(0)
    var = ((z * z).mean(0) - m * m).clamp_min(0)
    eps = float(np.float32(1e-5))
    inv = 1.0 / torch.sqrt(var + eps)
    xh = (z - m) * inv
    gam, bet = S["pre"]["bn4.weight"].double(), S["pre"]["bn4.bias"].double()
    v = xh * gam + bet
    lse = torch.logsumexp(v, 1)
    loss = (lse - v.gather(1, lab[:, None])[:, 0]).mean()
    p = torch.softmax(v, 1)
    dv = (p - F.one_hot(lab, 10).double()) / B
    db, dg = dv.sum(0), (dv * xh).sum(0)
    d = gam * inv * (dv - db / B - xh * dg / B)
    # fp32 softmax of |v| <~ 10: exp and the division a few ulp of p; mean / invstd rounded to fp32 (xh within 2^-22 |xh| + ...)
    tol_d = 2.0 ** -17 * (gam * inv).abs() * (p / B + dv.abs() + db.abs() / B + (xh * dg).abs() / B) + 1e-30
    R.within("head.loss", S["loss"][0], loss, 2.0 ** -18 * (loss.abs() + lse.abs().mean()))
    R.within("head.g4", S["g4"], d, tol_d)
    R.exact("head.gyp4", S["gyp4"][:, :10], S["g4"].to(torch.bfloat16))
    R.exact("head.gyp4.pad", S["gyp4"][:, 10:].float(), torch.zeros(B, 6, device=z.device))
    R.within("head.dbeta", S["grad"]["bn4.bias"], db, 2.0 ** -17 * (dv.abs().sum(0) + p.sum(0) / B))
    R.within("head.dgamma", S["grad"]["bn4.weight"], dg, 2.0 ** -17 * ((dv * xh).abs().sum(0) + (p * xh.abs()).sum(0) / B))
    mom = float(np.float32(0.1))
    rm0, rv0 = S["pre_bn"]["bn4"]
    rm, rv = S["bn"]["bn4"]
    rmr, rvr = (1 - mom) * rm0.double() + mom * m, (1 - mom) * rv0.double() + mom * var * B / (B - 1)
    R.within("bn4.running_mean", rm, rmr, _ulp(rmr))
    R.within("bn4.running_var", rv, rvr, _ulp(rvr))


def _gy_nchw(S, key, C_):
    gy = S[key]
    if gy.dim() == 2:
        return gy[:, :C_].double()[:, :, None, None]
    return gy[..., :C_].permute(0, 3, 1, 2).double()


def _gy1(S, R):
    """conv1's grad_output from the planes layout on the 32 x 32 grid: [B, 65, 28, 28]; zeros elsewhere"""
    B = S["E"]["B"]
    stride = (B * 1024 + 127) // 128 * 128
    pl = S["gyp1"].reshape(-1)[:9 * stride * 8].reshape(9, stride, 8)
    full = pl[:, :B * 1024].reshape(9, B, 32, 32, 8).permute(1, 0, 4, 2, 3).reshape(B, 72, 32, 32).double()
    outside = full.clone()
    outside[:, :65, :28, :28] = 0
    R.exact("gyp1.outside", outside, torch.zeros_like(outside))
    return full[:, :65, :28, :28]


def check_wgrads(S, R):
    E, eng, B = S["E"], S["eng"], S["E"]["B"]
    wg = [args[0] for args in _calls(S, "nn_noisy_conv_wgrad")]
    spec = [(3, "xp4", 390, "gyp4", 10), (2, "xp3", 120, "gyp3", 390), (1, "xp2", 65, "gyp2", 120), (0, "xp1", 3, None, 65)]
    for a, (li, xk, cin, gk, cout) in zip(wg, spec):
        name = WEIGHTS[li]
        R.true("wgrad.%s.args" % name, a.x_packed == getattr(eng, xk).data_ptr() and a.gw == S["m"].get_parameter(name).grad.data_ptr()
               and a.a_code_scale == np.float32(E["a_cs"][li]) and (a.w_lo, a.w_hi) == ((-1.0, 1.0) if E["q"] else (0.0, 0.0)), "arguments")
        x = _x_values(S, xk, cin)
        gy = _gy1(S, R) if gk is None else _gy_nchw(S, gk, cout)
        shape = _w_main(S, li).shape
        sc = E["a_cs"][li] or 1.0
        ref = torch.nn.grad.conv2d_weight(x, shape, gy) * sc
        n = B * gy.shape[2] * gy.shape[3]
        tol = n * U24 * torch.nn.grad.conv2d_weight(x.abs(), shape, gy.abs()) * sc + 2.0 ** -23 * ref.abs() + 1e-30
        if E["q"]:
            keep = (S["pre"][name].abs() <= 1.0).reshape(shape)
            ref = torch.where(keep, ref, torch.zeros_like(ref))
        R.within("wgrad.%s" % name, S["grad"][name].reshape(shape), ref, tol)


def check_dgrads(S, R):
    E, eng, B = S["E"], S["eng"], S["E"]["B"]
    dg = [args[0] for args in _calls(S, "nn_noisy_conv_dgrad")] + [args[0] for args in _calls(S, "nn_conv_dgrad_planes")]
    spec = [(3, "gyp4", 10, "gx4", (B, 390, 1, 1)), (2, "gyp3", 390, "gx3", (B, 120, 5, 5)), (1, "gyp2", 120, "gx2", (B, 65, 14, 14))]
    for a, (li, gk, cout, ok, xshape) in zip(dg, spec):
        R.true("dgrad.%s.args" % ok, a.gy_packed == getattr(eng, gk).data_ptr() and a.gx == getattr(eng, ok).data_ptr()
               and a.w_code_scale == np.float32(E["w_cs"]) and a.w_packed == eng.wp_dgrad[li], "arguments")
        gy = _gy_nchw(S, gk, cout)
        wm = _w_main(S, li)
        sc = E["w_cs"] or 1.0
        ref = torch.nn.grad.conv2d_input(xshape, wm, gy) * sc
        n = wm.shape[0] * wm.shape[2] * wm.shape[3]
        tol = n * U24 * torch.nn.grad.conv2d_input(xshape, wm.abs(), gy.abs()) * sc + 2.0 ** -23 * ref.abs() + 1e-30
        R.within("dgrad.%s" % ok, S[ok].reshape(xshape), ref, tol)


def _bwd_one(S, R, name, sb, g, x, amax, C_, H, pool, key, act_max, q_hi, gy_planes=False):
    """one stage backward: masks exact (both FMA contractions agree), dgamma / dbeta, and the packed gradient within the
    bf16 images of [D - tol, D + tol] (tol of the stage sweep's fp32 formula)"""
    E, B = S["E"], S["E"]["B"]
    PH = H // 2 if pool else H
    mean, invstd = S["stat"][key]
    gam, bet = S["pre"][key + ".weight"], S["pre"][key + ".bias"]
    qh = q_hi if E["q"] else float("inf")
    args = (x.reshape(B, C_, -1).cpu().numpy(), g.reshape(B, C_, -1).cpu().numpy(), mean.cpu().numpy(), invstd.cpu().numpy(),
            gam.cpu().numpy(), bet.cpu().numpy(), act_max, qh)
    dv0, xhat, _ = _bwd_reference(*args)
    dv1, _, _ = _bwd_reference(*args, fma=True)
    amb = torch.from_numpy(dv0 != dv1).to(g.device)
    dv, xh = torch.from_numpy(dv0).double().to(g.device), torch.from_numpy(xhat).double().to(g.device)
    gabs = g.reshape(B, C_, -1).double().abs()
    db_ref, dgm_ref = dv.sum((0, 2)), (dv * xh).sum((0, 2))
    amb_db, amb_dg = (gabs * amb).sum((0, 2)), (gabs * xh.abs() * amb).sum((0, 2))
    R.within(name + ".dbeta", S["grad"][key + ".bias"], db_ref, 2.0 ** -22 * dv.abs().sum((0, 2)) + amb_db + 1e-30)
    R.within(name + ".dgamma", S["grad"][key + ".weight"], dgm_ref, 2.0 ** -22 * (dv * xh).abs().sum((0, 2)) + amb_dg + 1e-30)
    ic = float(np.float32(1.0) / (np.float32(B) * np.float32(PH) * np.float32(PH)))
    e = lambda t: t.double()[None, :, None]
    a_ = e(S["grad"][key + ".bias"]) * ic
    q_ = xh * e(S["grad"][key + ".weight"]) * ic
    gi = e(gam) * e(invstd)
    D = gi * (dv - a_ - q_)
    tol = 2.0 ** -21 * gi.abs() * (dv.abs() + a_.abs() + q_.abs()) + 1e-30
    lo, hi = (D - tol).to(torch.bfloat16).double(), (D + tol).to(torch.bfloat16).double()
    if pool:
        am = amax.reshape(B, C_, PH, PH).long()
        got = gy_planes if gy_planes is not False else _gy_nchw(S, name_to_gyp(name), C_)
        win = got.reshape(B, C_, PH, 2, PH, 2).permute(0, 1, 2, 4, 3, 5).reshape(B, C_, PH, PH, 4)
        sel = win.gather(-1, am[..., None])[..., 0].reshape(B, C_, -1)
        others = win.clone()
        others.scatter_(-1, am[..., None], 0.0)
        R.exact(name + ".routing", others, torch.zeros_like(others))
    else:
        sel = _gy_nchw(S, name_to_gyp(name), C_).reshape(B, C_, -1)
    ok = ((sel >= lo) & (sel <= hi)) | amb
    R.exact(name + ".gy", ok, torch.ones_like(ok))
    R.true(name + ".ambiguous", float(amb.double().mean()) < 1e-4, "%d elements depend on the FMA contraction" % int(amb.sum()))


def name_to_gyp(name):
    return {"bwd3": "gyp3", "bwd2": "gyp2", "bwd1": "gyp1"}[name]


def check_stage_bwd(S, R):
    E, eng = S["E"], S["eng"]
    am, qh = E["act_max"], E["q_hi"]
    sb = [args[0] for args in _calls(S, "nn_stage_bwd")]
    for a, (name, g, x, key, gyp, act, q) in zip(sb, [("bwd3", eng.gx4, eng.l1n, "bn3", eng.gyp3, am[2], qh[3]),
                                                     ("bwd2", eng.gx3, eng.pool2, "bn2", eng.gyp2, am[1], qh[2]),
                                                     ("bwd1", eng.gx2, eng.pool1, "bn1", eng.gyp1, am[0], qh[1])]):
        R.true(name + ".args", a.g == g.data_ptr() and a.x == x.data_ptr() and a.gyp == gyp.data_ptr() and a.act_max == np.float32(act)
               and a.q_hi == q and a.q_bits == E["q"] and a.mean == eng.stat[key][0].data_ptr(), "arguments")
    _bwd_one(S, R, "bwd3", sb[0], S["gx4"], S["l1n"], None, 390, 1, 0, "bn3", am[2], qh[3])
    _bwd_one(S, R, "bwd2", sb[1], S["gx3"], S["pool2"], S["amax2"], 120, 10, 1, "bn2", am[1], qh[2])
    _bwd_one(S, R, "bwd1", sb[2], S["gx2"], S["pool1"], S["amax1"], 65, 28, 1, "bn1", am[0], qh[1], gy_planes=_gy1(S, R))


def check_adamw(S, R):
    opt = S["opt"]
    parts = _calls(S, "step_part")
    R.true("adamw.parts", [p[1] for p in parts] == [False, True] and sorted(parts[0][0] + parts[1][0]) == sorted(S["pre"])
           and set(parts[0][0]) == {"linear2.weight", "linear1.weight", "conv2.weight"}, "partition %r" % [p[0] for p in parts])
    b1, b2 = (float(np.float32(b)) for b in opt.param_groups[0]["betas"])         # the kernel takes fp32 betas
    eps = float(np.float32(opt.param_groups[0]["eps"]))
    t = S["pre_step"] + 1
    bc1 = float(np.float32(1.0 - b1 ** t))
    bc2s = float(np.float32(math.sqrt(1.0 - b2 ** t)))
    names = {id(p): n for n, p in S["m"].named_parameters()}
    for i, (grp, p) in enumerate(opt._params()):
        n = names[id(p)]
        lr, wd, clamp = float(np.float32(grp["lr"])), float(np.float32(grp["weight_decay"])), float(np.float32(grp["clamp"]))
        step_size = float(np.float32(lr / bc1))
        g = S["grad"][n].double() * opt.grad_scale
        p0, m0, v0 = S["pre"][n].double(), S["pre_m"][n].double(), S["pre_v"][n].double()
        decay = float(np.float32(1.0 - np.float32(lr) * np.float32(wd)))
        m = m0 + (1 - b1) * (g - m0)
        v = v0 * b2 + (1 - b2) * g * g
        denom = torch.sqrt(v) / bc2s + eps
        upd = step_size * m / denom
        w = p0 * decay - upd
        if clamp > 0:
            w = w.clamp(-clamp, clamp)
        tol = 2.0 ** -21 * (p0.abs() + step_size * (m0.abs() + g.abs()) / denom) + 1e-30
        R.within("adamw.%s" % n, S["post"][n], w, tol)
        R.within("adamw.%s.exp_avg" % n, S["post_m"][n], m, 2.0 ** -22 * (m0.abs() + g.abs()) + 1e-30)
        R.true("adamw.%s.absmax" % n, float(S["absmax"][i]) == float(S["post"][n].abs().max()), "absmax")


CHECKS = [check_coverage, check_weight_codes, check_input_pack, check_conv1, check_stage_fwd, check_fwd_gemms, check_head,
          check_wgrads, check_dgrads, check_stage_bwd, check_adamw]


def run_checks(S, checks=CHECKS):
    R = Report()
    for c in checks:
        c(S, R)
    return R


# ---------------------------------------------------------------------------------------------- CPU tests

def test_philox_port_matches_oracle():
    from oracle.noisynet_oracle import philox4x32_10, philox_normal_mn
    g = np.array([0, 1, 2, 3, 2 ** 32 - 1, 2 ** 32, 123456789012, 2 ** 40 + 5], dtype=np.uint64)
    for seed, off in ((0, 0), (0x5EED1234ABCD, 77), (2 ** 64 - 1, 2 ** 40 + 3)):
        want = philox4x32_10(g, seed, off).astype(np.int64)
        got = _philox_t(torch.from_numpy(g.astype(np.int64)), seed, off).numpy()
        assert np.array_equal(got, want)
    z = _normal_mn_t(7, 13, 4242, 17, "cpu").numpy()
    assert np.abs(z - philox_normal_mn(7, 13, 4242, 17)).max() <= 1e-6       # float64 libm differences only


def test_restatements_detect_one_off():
    """the weight quantizer and the input pack restatements against an independent float32 evaluation of the spec
    (oracle.philox_uniform_sym, stage sweep mapping), and a one-off code is seen"""
    from oracle.noisynet_oracle import philox4x32_10, philox_uniform_sym
    gen = torch.Generator().manual_seed(5)
    w = torch.randn(37, 5, 3, generator=gen) * 0.5
    w[0, 0, 0] = 1.5                                       # clipped
    seed, off = 0x1234, 88
    got = weight_codes(w, 4, 1.0, 0.5, seed, off).reshape(w.shape)
    u = torch.from_numpy(philox_uniform_sym(w.numel(), seed, off, 0.5)).reshape(w.shape)
    s = np.float32(2.0 / 15.0)
    t = ((w + 1.0) / torch.tensor(s) + u).clamp(0, 15)
    want = (2 * torch.round(t) - 15).to(torch.int8)
    assert torch.equal(got, want)
    bad = want.clone()
    bad[3, 2, 1] += 2
    assert not torch.equal(got, bad)
    x = torch.rand(2, 3, 4, 5, generator=gen)
    got = input_codes(x, 4, 1.0, 0.5, seed, off)
    pix = np.arange(2 * 20, dtype=np.uint64)
    r = philox4x32_10(np.stack([2 * pix, 2 * pix + 1], -1), seed, off).reshape(40, 8)[:, :3]
    uu = ((r >> np.uint32(8)).astype(np.float32) * np.float32(2.0 ** -24) * np.float32(1.0) - np.float32(0.5))
    uu = torch.from_numpy(uu).reshape(2, 4, 5, 3).permute(0, 3, 1, 2)
    want = torch.round((x / torch.tensor(np.float32(1.0 / 15.0)) + uu).clamp(0, 15))
    assert torch.equal(got, want)
    want[1, 2, 3, 4] += 1
    assert not torch.equal(got, want)


def test_report_bounds_fail():
    R = Report()
    R.within("a", torch.tensor([1.0, 2.0]), torch.tensor([1.0, 2.0], dtype=torch.float64), torch.full((2,), 1e-6, dtype=torch.float64))
    assert not R.bad
    R.within("b", torch.tensor([1.0, 2.1]), torch.tensor([1.0, 2.0], dtype=torch.float64), torch.full((2,), 1e-6, dtype=torch.float64))
    R.exact("c", torch.tensor([1, 2]), torch.tensor([1, 3]))
    assert len(R.bad) == 2


# ---------------------------------------------------------------------------------------------- GPU tests

@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    torch.backends.cudnn.allow_tf32 = False
    torch.backends.cuda.matmul.allow_tf32 = False
    return torch.device("cuda:0")


_KEEP = {}


@pytest.mark.gpu
@pytest.mark.parametrize("cid", list(CONFIGS))
def test_step_launches(dev, cid):
    S = run_step(dev, cid)
    R = run_checks(S)
    print("\n%s: check, max |error|, bound at the worst element, worst error / bound" % cid)
    for name, err, tol, ratio in R.rows:
        print("  %-34s %.3e  %.3e  %.3g" % (name, err, tol, ratio))
    if cid == "q4-512":
        _KEEP[cid] = S
    assert not R.bad, "\n".join(R.bad)


def _perturbed(S, key, fn, sub=None):
    T = dict(S)
    if sub is None:
        T[key] = S[key].clone()
        fn(T[key])
    else:
        T[key] = dict(S[key])
        T[key][sub] = tuple(t.clone() for t in S[key][sub]) if isinstance(S[key][sub], tuple) else S[key][sub].clone()
        fn(T[key][sub])
    return T


def _recorded(S, name, idx, edit):
    """S with the idx-th call of `name` given edited argument snapshots"""
    T = dict(S)
    calls, k = [], 0
    for n, args in S["calls"]:
        if n == name:
            if k == idx:
                args = [type(a).from_buffer_copy(a) if isinstance(a, (C.Structure, C.Array)) else a for a in args]
                edit(args)
            k += 1
        calls.append((n, args))
    T["calls"] = calls
    return T


def _set(i, field, value):
    def edit(args):
        setattr(args[i], field, value)
    return edit


def _bump(t):
    k = t.numel() // 3
    t.view(-1)[k] += 1 if not t.is_floating_point() else max(1e-2, 1e-2 * abs(float(t.view(-1)[k])))


@pytest.mark.gpu
def test_checks_detect_one_change(dev):
    """every check raises on its q4-512 step with one output element moved, or one recorded argument changed"""
    S = _KEEP.get("q4-512") or run_step(dev, "q4-512")
    assert not run_checks(S).bad
    cases = [
        (check_coverage, dict(S, calls=S["calls"][:-1])),
        (check_weight_codes, _perturbed(S, "wcodes", _bump, 2)),
        (check_weight_codes, _recorded(S, "nn_prepare_weights", 1, lambda a: setattr(a[0][0].rng, "offset", a[0][0].rng.offset + 4))),
        (check_input_pack, _perturbed(S, "x1_planes", _bump)),
        (check_conv1, _perturbed(S, "pool1", _bump)),
        (check_conv1, _perturbed(S, "stat", lambda t: t[0].view(-1)[5].add_(1e-3 + 1e-2 * abs(float(t[0][5]))), "bn1")),
        (check_conv1, _recorded(S, "nn_noisy_conv_fwd", 0, _set(0, "a_code_scale", 2.0 / 15.0))),
        (check_stage_fwd, _perturbed(S, "xp3", lambda t: t.view(-1)[7].add_(1))),
        (check_stage_fwd, _recorded(S, "nn_stage_fwd", 0, _set(0, "act_max", 4.5))),
        (check_stage_fwd, _recorded(S, "nn_stage_fwd", 2, _set(0, "q_hi", 4.0))),
        (check_stage_fwd, _perturbed(S, "xmax2", lambda t: t.mul_(1 + 2 ** -20))),
        (check_fwd_gemms, _perturbed(S, "y2n", _bump)),
        (check_fwd_gemms, _perturbed(S, "l1n", _bump)),
        (check_fwd_gemms, _recorded(S, "nn_noisy_conv_fwd", 3, lambda a: setattr(a[0].rng, "offset", a[0].rng.offset + 4))),
        (check_head, _perturbed(S, "g4", _bump)),
        (check_head, _perturbed(S, "gyp4", lambda t: t.view(-1)[3].mul_(2))),
        (check_wgrads, _perturbed(S, "grad", _bump, "conv2.weight")),
        (check_wgrads, _perturbed(S, "grad", lambda t: t.view(-1)[5].add_(1.0), "conv1.weight")),
        (check_dgrads, _perturbed(S, "gx3", _bump)),
        (check_stage_bwd, _perturbed(S, "gyp2", lambda t: t.view(-1)[int((t.view(-1) != 0).nonzero()[0, 0])].mul_(2))),
        (check_stage_bwd, _recorded(S, "nn_stage_bwd", 1, _set(0, "act_max", 4.0))),
        (check_adamw, _perturbed(S, "post", _bump, "linear1.weight")),
        (check_adamw, _perturbed(S, "grad", lambda t: t.view(-1)[11].add_(1e-3), "conv2.weight")),
    ]
    missed = [i for i, (check, T) in enumerate(cases) if not run_checks(T, [check]).bad]
    assert not missed, "checks that did not notice: %s" % [cases[i][0].__name__ for i in missed]
