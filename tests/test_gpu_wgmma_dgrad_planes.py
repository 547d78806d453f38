"""The dgrad on a resident row-plane image of grad_output (k_dgrad_planes, csrc/nn_conv_tma.cu; nn_conv_dgrad_planes).

It reads each grad_output image once and takes all taps from shared memory, but it runs the same k16 groups in the same
order as k_conv_tma<2, NT> (nn_noisy_conv_dgrad), so its gx is expected to be bit-identical to that kernel's, and, on the
exact integer operands of test_gpu_tma_sweep.py, bit-identical to float64.  Every GPU case asserts under torch.profiler
which kernel ran.
"""
import copy
import ctypes as C
import re

import numpy as np
import pytest
import torch

from test_gpu_tma_sweep import _exact, _grads, _nhwc_bf16, _scaled, _w_raw, tma_plan

NONE = 0
_KERNEL = re.compile(r"\b(k_dgrad_planes|k_conv_tma|k_conv_umma)\b(<[^>]*>)?")


def _geom(B, cin, H, cout, k, stride=1, pad=0, W=None):
    from noisynet_b200._lib import ConvGeom
    return ConvGeom(B, cin, H, H if W is None else W, cout, k, k if W is None else k, stride, pad)


# ---------------------------------------------------------------------------------------------- CPU tests

@pytest.fixture(scope="module")
def lib():
    import __graft_entry__ as entry
    entry.build()
    from noisynet_b200 import _lib
    return _lib.load()


def test_query_serves_conv2_and_refuses_outside_its_limits(lib):
    ok = lambda g: lib.nn_conv_dgrad_planes_ok(C.byref(g))
    assert ok(_geom(512, 65, 14, 120, 5)) == 1                   # NoisyNet conv2: 14 x 18 virtual rows
    assert ok(_geom(1, 65, 14, 120, 5)) == 1
    assert ok(_geom(3, 16, 10, 16, 3, pad=1)) == 1
    assert ok(_geom(512, 65, 14, 120, 5, stride=2)) == 0         # stride 2
    assert ok(_geom(512, 65, 14, 136, 5)) == 0                   # > 128 grad_output channels
    assert ok(_geom(512, 121, 14, 120, 5)) == 0                  # > 120 columns: two n-tiles
    assert ok(_geom(512, 65, 16, 120, 5)) == 0                   # 16 x 20 virtual rows > 256
    assert ok(_geom(512, 64, 32, 64, 3, pad=1)) == 0             # ResNet 3x3 layers
    assert ok(_geom(512, 128, 16, 128, 3, pad=1)) == 0
    assert ok(_geom(512, 65, 14, 120, 5, pad=5)) == 0            # pad >= K
    assert ok(_geom(512, 65, 14, 8, 5)) == 0                     # 8 channels: the plan of the shift kernels


class _Recorder:
    def __init__(self):
        self.calls = []

    def __getattr__(self, name):
        def call(*args):
            self.calls.append(name)
            return 0
        return call


@pytest.mark.parametrize("planes", [True, False])
def test_engine_routes_conv2_dgrad(planes):
    """NoisyNetEngine._dgrad calls nn_conv_dgrad_planes for conv2 when the query served it, nn_noisy_conv_dgrad otherwise
    and for every other layer"""
    from types import SimpleNamespace

    from noisynet_b200.engine import NoisyNetEngine
    rec = _Recorder()
    eng = SimpleNamespace(lib=rec, dgrad_planes=planes, wp_dgrad={1: 0, 2: 0}, wp_dgrad_layout={1: 2, 2: 0}, w_cs={1: 1.0, 2: 1.0},
                          ws=torch.zeros(16, dtype=torch.uint8), di=0, _st=lambda: None)
    t = torch.zeros(4)
    NoisyNetEngine._dgrad(eng, _geom(2, 65, 14, 120, 5), t, 1, t)
    NoisyNetEngine._dgrad(eng, _geom(2, 3000, 1, 1, 390), t, 2, t)
    assert rec.calls == ["nn_conv_dgrad_planes" if planes else "nn_noisy_conv_dgrad", "nn_noisy_conv_dgrad"]


# ---------------------------------------------------------------------------------------------- GPU plumbing

@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available()
    import __graft_entry__ as entry
    entry.build()
    return torch.device("cuda:0")


def _seen(fn):
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
    return out, seen


def _launch(expect, fn):
    """fn under torch.profiler: the conv kernels it launched are exactly `expect` (profiled again, up to three times in
    all, if the profiler missed the launch: the routing is deterministic, so a wrong kernel fails every time)"""
    from noisynet_b200 import ops
    for _ in range(3):
        out, seen = _seen(fn)
        if seen == set(expect):
            break
    assert ops.error_flag() == 0
    assert seen == set(expect), (sorted(seen), sorted(expect))
    return out


class Packed:
    """a layer's NN_PACK_TMA dgrad image from nn_prepare_weights (4-bit round-to-nearest codes, as the engine packs it)"""

    def __init__(self, dev, cout, cin, k, gen):
        from noisynet_b200 import _lib
        from noisynet_b200._lib import PACK_TMA, Rng, WPrepJob
        from oracle import noisynet_oracle as O
        self.lib = lib = _lib.load()
        wr = _w_raw((cout, cin, k, k), gen)
        self.w_cs = float(np.float32(2.0 / 15.0)) / 2.0
        wq = O.uniform_quantize_fwd(wr, 4, -1.0, 1.0)
        self.codes = torch.round(wq.double() / self.w_cs)
        self.wr = wr.to(dev)
        self.scratch = torch.zeros(wr.numel() + 16, dtype=torch.int8, device=dev)
        jb = self.job = (WPrepJob * 1)()
        j = jb[0]
        j.w_raw = self.wr.data_ptr()
        j.Cout, j.Cin, j.KHW, j.mode, j.m_rows, j.noise_mode, j.want_wsum = cout, cin, k * k, 1, 1, NONE, 0
        j.layout, j.q_bits, j.q_hi, j.stochastic, j.u_inject, j.rng = PACK_TMA, 4, 1.0, 0.0, None, Rng(0, 0, None)
        j.codes = self.scratch.data_ptr()
        self.buf = torch.zeros(int(lib.nn_weight_pack_bytes(C.byref(j))) + 1024, dtype=torch.uint8, device=dev)
        j.packed_out = (self.buf.data_ptr() + 1023) // 1024 * 1024
        _lib.check(lib.nn_prepare_weights(jb, 1, 0, torch.cuda.current_stream().cuda_stream), "nn_prepare_weights")


def _dgrad(pk, geom, gyp, gx, planes):
    from noisynet_b200 import _lib
    from noisynet_b200._lib import PACK_TMA, PREC_BF16, ConvDgradArgs
    ws = torch.empty(int(pk.lib.nn_conv_workspace_bytes(C.byref(geom), PREC_BF16)) + 4096, dtype=torch.uint8, device=gx.device)
    d = ConvDgradArgs()
    d.g, d.gy, d.w_eff, d.gx, d.precision, d.w_code_scale = geom, None, None, gx.data_ptr(), PREC_BF16, pk.w_cs
    d.workspace, d.workspace_bytes = ws.data_ptr(), ws.numel()
    d.gy_packed, d.w_packed, d.w_packed_layout = gyp.data_ptr(), pk.job[0].packed_out, PACK_TMA
    st = torch.cuda.current_stream().cuda_stream
    if planes:
        _lib.check(pk.lib.nn_conv_dgrad_planes(C.byref(d), 0, st), "nn_conv_dgrad_planes")
    else:
        _lib.check(pk.lib.nn_noisy_conv_dgrad(C.byref(d), 0, st), "nn_noisy_conv_dgrad")
    return gx


def _run(pk, geom, gyp, shape, planes, nt):
    gx = torch.full(shape, float("nan"), device=gyp.device)
    name = "k_dgrad_planes<%d>" % nt if planes else "k_conv_tma<2, %d>" % nt
    return _launch({name}, lambda: _dgrad(pk, geom, gyp, gx, planes))


# ---------------------------------------------------------------------------------------------- GPU tests
# layer (B, Cin, H, Cout, k, pad): conv2 at four batches (odd ones: a CTA that reloads its partner's image), then other
# widths: 16-channel tail only, one 64-channel chunk, 64 + 16, two chunks; n-tiles of 8 .. 120 columns
EXACT = [(1, 65, 14, 120, 5, 0), (3, 65, 14, 120, 5, 0), (6, 65, 14, 120, 5, 0), (512, 65, 14, 120, 5, 0),
         (5, 16, 10, 16, 3, 1), (4, 120, 12, 64, 3, 0), (3, 8, 9, 72, 2, 1), (7, 33, 11, 128, 4, 2), (300, 65, 14, 120, 5, 0)]


@pytest.mark.gpu
@pytest.mark.parametrize("case", EXACT, ids=lambda c: "B%d-%d-%d-%d-k%d-p%d" % c)
def test_exact_integer_operands(dev, case):
    B, cin, H, cout, k, pad = case
    assert _plan_ok(B, cin, H, cout, k, pad)
    nt = tma_plan(cout, k, cin, False)["n_t"]
    gen = torch.Generator().manual_seed(sum(case))
    OH = H + 2 * pad - k + 1
    pk = Packed(dev, cout, cin, k, gen)
    gy = _grads((B, cout, OH, OH), gen)
    gyp = _nhwc_bf16(gy.to(dev), (cout + 7) // 8 * 8)
    geom = _geom(B, cin, H, cout, k, pad=pad)
    gx = _run(pk, geom, gyp, (B, cin, H, H), True, nt)
    r = _exact(torch.nn.grad.conv2d_input((B, cin, H, H), pk.codes.to(dev), gy.to(dev).double(), 1, pad))
    assert torch.equal(gx, _scaled(r, pk.w_cs))


def _plan_ok(B, cin, H, cout, k, pad):
    from noisynet_b200 import _lib
    return _lib.load().nn_conv_dgrad_planes_ok(C.byref(_geom(B, cin, H, cout, k, pad=pad))) == 1


@pytest.mark.gpu
@pytest.mark.parametrize("B", [3, 512])
def test_bit_identical_to_tma_conv_dgrad(dev, B):
    """non-integer bf16 gradients on conv2's packed image: gx equals k_conv_tma<2, 72>'s bit for bit, run after run"""
    gen = torch.Generator().manual_seed(600 + B)
    pk = Packed(dev, 120, 65, 5, gen)
    gy = torch.randn(B, 120, 10, 10, generator=gen) * 3e-3
    gyp = _nhwc_bf16(gy.to(dev), 120)
    geom = _geom(B, 65, 14, 120, 5)
    ref = _run(pk, geom, gyp, (B, 65, 14, 14), False, 72)
    got = [_run(pk, geom, gyp, (B, 65, 14, 14), True, 72) for _ in range(2)]
    assert torch.isfinite(ref).all() and ref.abs().max().item() > 0
    assert torch.equal(got[0], ref)
    assert torch.equal(got[0], got[1])


@pytest.mark.gpu
def test_refused_call_fails_loudly(dev):
    from noisynet_b200._lib import NoisyNetLibraryError
    gen = torch.Generator().manual_seed(7)
    pk = Packed(dev, 120, 65, 5, gen)
    gyp = torch.zeros(2, 10, 10, 120, dtype=torch.bfloat16, device=dev)
    gx = torch.zeros(2, 65, 14, 14, device=dev)
    with pytest.raises(NoisyNetLibraryError, match="not served"):
        _dgrad(pk, _geom(2, 65, 14, 120, 5, stride=2), gyp, gx, True)


class _Calls:
    """the engine's library handle, recording which entry points a step calls"""

    def __init__(self, lib):
        self._lib, self.names = lib, []

    def __getattr__(self, name):
        self.names.append(name)
        return getattr(self._lib, name)


@pytest.mark.gpu
def test_engine_step_routes_conv2_dgrad_and_matches_tma_dgrad(dev):
    """one training step of the benchmark configuration runs conv2's dgrad through nn_conv_dgrad_planes (whose kernel the
    tests above pin under the profiler), and every gradient equals that of an engine routed through nn_noisy_conv_dgrad,
    bit for bit (same injected draws).  The step itself is not profiled: a profiled multi-stream training step leaves
    torch.profiler missing kernels in the later sessions of a long test process."""
    from noisynet_b200 import ops
    from noisynet_b200.engine import NoisyNetEngine
    from noisynet_b200.net import NoisyNet, default_args, with_quant
    from oracle import noisynet_oracle as O
    from test_gpu_net import _make_rnd
    B, q = 512, 4
    oa = O.default_args(q_a=q, q_w=q, quant_max2=5.0, quant_max4=5.0, current=1.0)
    torch.manual_seed(11)
    na = with_quant(default_args(layer_currents=[1.0] * 4), q, q)
    ms = [NoisyNet(na, fused=True, precision="bf16").to(dev)]
    ms[0].quantize2.running_max = torch.tensor(5.0, device=dev)       # calibrated activation ranges, as in the benchmark
    ms[0].quantize4.running_max = torch.tensor(5.0, device=dev)
    ms.append(copy.deepcopy(ms[0]))
    engs = [NoisyNetEngine(m, B, opt=None) for m in ms]
    assert engs[0].dgrad_planes
    engs[1].dgrad_planes = False
    x, lab = O.synthetic_cifar(B, seed=21)
    rnd = _make_rnd(oa, B, q, 301)
    calls = []
    for e in engs:
        for m in e.m.parameters():
            m.grad.zero_()
        e.inject = dict(u=[rnd[k].to(dev) for k in ("ua1", "ua2", "ua3", "ua4")],
                        uw=[rnd[k].to(dev) for k in ("uw0", "uw1", "uw2", "uw3")],
                        z=[rnd[k].to(dev) for k in ("z0", "z1", "z2", "z3")])
        e.lib = _Calls(e.lib)
        e.train_step(x.to(dev), lab.to(dev))
        torch.cuda.synchronize()
        calls.append(e.lib.names)
        e.lib = e.lib._lib
        assert ops.error_flag() == 0
    assert calls[0].count("nn_conv_dgrad_planes") == 1 and calls[0].count("nn_noisy_conv_dgrad") == 2, calls[0]
    assert "nn_conv_dgrad_planes" not in calls[1] and calls[1].count("nn_noisy_conv_dgrad") == 3, calls[1]
    assert torch.equal(engs[0].gx2, engs[1].gx2)
    for (k, a), b in zip(ms[0].named_parameters(), ms[1].parameters()):
        assert torch.equal(a.grad, b.grad), k
