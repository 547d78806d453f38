"""NoisyNetEngine -- the whole CIFAR NoisyNet training step (noisynet.py:1276-1542) as an explicit schedule
of this library's kernels, with static buffers (CUDA-graph capturable, no autograd, no torch kernels):

  forward : input quantize+pack -> [tensor-core fused noisy conv -> pool+BN+ReLU+clamp+dropout+quantize+pack stage] x 2
            -> [tensor-core fused noisy linear -> BN+ReLU+clamp+dropout+quantize+pack stage] -> fused noisy linear -> BN + CE head
  backward: head -> wgrad/dgrad (tensor cores) -> stage backward (STE/dropout/clamp/ReLU masks, BN backward, pool routing,
            emitted as NHWC bf16 for the next wgrad/dgrad) ... -> conv1 wgrad
  update  : [flat-gradient all-reduce] -> fused AdamW + weight clamp + max|W|

Activations travel between layers as NHWC bf16 integer codes (exact 4-bit operands for the tensor cores);
fp32 NCHW tensors exist only where the maths needs them (noisy conv outputs, pooled BN inputs, gradients).
Parameters, BN buffers and quantizer ranges are those of a `NoisyNet` module (state_dict compatible).
Per-layer bit widths (q = 0: bf16 operands) and act_max1..3 are honoured; steady-state semantics (the i < 20 side
statistics, bias and the alternative noise models are the module path's).  --dropout p (noisynet.py:375-376) runs inside
the stage kernels at the reference's sites -- after relu2 and relu3, and after relu1 when --dropout_conv > 0 (at rate
--dropout, as the reference does) -- with a Bernoulli keep mask drawn in the forward kernel and reused by the backward.
``eval_forward`` is the model.eval() forward (running BN statistics, no stochastic rounding, no dropout, noise still
injected).
"""
import ctypes as C
import os

import torch

from . import _lib, ops
from ._lib import (NOISE_EXTERNAL, NOISE_MERGED, PACK_SHIFT, PACK_TMA, PREC_BF16, ConvDgradArgs, ConvFwdArgs, ConvGeom, ConvWgradArgs,
                   Rng, StageArgs, StageBwdArgs, TailArgs, WPrepJob)
from .hardware_model import _f32


def _p(t):
    return None if t is None else t.data_ptr()


class _Layer:
    pass


class NoisyNetEngine:
    def __init__(self, model, batch, opt=None, reducer=None):
        a = model.args
        self.q_w = [int(a.q_w1), int(a.q_w2), int(a.q_w3), int(a.q_w4)]          # per-layer weight bits (noisynet.py:898-900)
        self.q_a = [int(a.q_a1), int(a.q_a2), int(a.q_a3), int(a.q_a4)]
        # q = 0 on a layer (the README flags, noisynet.py:282-283): its operands travel as bf16-ROUNDED values instead of
        # exact integer codes (bf16 training tolerance 1.5e-2, fp32 accumulation), same kernels, scale factors 1
        if any(getattr(a, k, 0) > 0 for k in ("n_w1", "n_w2", "n_w3", "n_w4")) and min(self.q_w) == 0:
            raise NotImplementedError("NoisyNetEngine: multiplicative weight noise (--n_w) is served by the module path")
        if max(self.q_w) > 7:
            raise ValueError("NoisyNetEngine: weight codes are int8 (q_w <= 7)")
        if a.use_bias:
            raise NotImplementedError("NoisyNetEngine: bias is served by the module path (net.NoisyNet(fused=True), or the "
                                      "unchanged script on the drop-in modules), not the engine")
        if not 0.0 <= float(a.dropout) < 1.0:
            raise ValueError("NoisyNetEngine: dropout must lie in [0, 1)")
        if any(getattr(a, k, 0) for k in ("distort_act", "uniform_ind", "uniform_dep", "normal_ind", "normal_dep")):
            raise NotImplementedError("NoisyNetEngine: alternative noise models are served by the module path")
        for li, mod in enumerate((model.conv1, model.conv2, model.linear1, model.linear2)):
            if self.q_w[li] == 0:
                continue
            qm = mod.quantize_weights
            # the engine quantizes weights on the fixed range [-1, 1] (hardware_model.py:323): a percentile-calibrated
            # weight range (--calculate_running flips every QuantMeasure, noisynet.py:1209) is the module path's business
            if qm.calculate_running or qm.min_value != -1.0 or qm.max_value != 1.0 or float(qm.running_min.reshape(-1)[0]) < 0:
                raise NotImplementedError("NoisyNetEngine: weight quantizers must be on the fixed range [-1, 1]")
        self.m, self.a, self.B = model, a, int(batch)
        self.opt, self.red = opt, reducer
        self.dev = model.conv1.weight.device
        self.di = self.dev.index if self.dev.index is not None else torch.cuda.current_device()
        self.lib = _lib.load()
        B, dev = self.B, self.dev
        f32 = lambda *s: torch.empty(*s, dtype=torch.float32, device=dev)
        bf16 = lambda *s: torch.zeros(*s, dtype=torch.bfloat16, device=dev)
        C1, C2, FC = a.fm1 * a.width, a.fm2 * a.width, a.fc * a.width
        fs = a.fs
        H1 = 32 - fs + 1                  # 28
        P1 = H1 // 2                      # 14
        H2 = P1 - fs + 1                  # 10
        P2 = H2 // 2                      # 5
        self.dims = (C1, C2, FC, H1, P1, H2, P2)
        c8 = lambda c: (c + 7) // 8 * 8
        # activations
        self.xp1 = bf16(B, 32, 32, 8)
        self.y1n = f32(B, C1, H1, H1); self.pool1 = f32(B, C1, P1, P1); self.amax1 = torch.empty(B, C1, P1, P1, dtype=torch.uint8, device=dev)
        self.xp2 = bf16(B, P1, P1, c8(C1)); self.xmax2 = f32(1)
        self.y2n = f32(B, C2, H2, H2); self.pool2 = f32(B, C2, P2, P2); self.amax2 = torch.empty(B, C2, P2, P2, dtype=torch.uint8, device=dev)
        self.xp3 = bf16(B, P2, P2, c8(C2))
        self.l1n = f32(B, FC); self.xp4 = bf16(B, c8(FC)); self.xmax4 = f32(1)
        self.l2n = f32(B, 10)
        self.stat = {k: (f32(c), f32(c)) for k, c in (("bn1", C1), ("bn2", C2), ("bn3", FC))}
        # gradients of activations
        self.g4 = f32(B, 10); self.gyp4 = bf16(B, 16)
        self.gx4 = f32(B, FC); self.gyp3 = bf16(B, c8(FC))
        self.gx3 = f32(B, C2, P2, P2); self.gyp2 = bf16(B, H2, H2, c8(C2))
        self.gx2 = f32(B, C1, P1, P1); self.gyp1 = bf16(B, H1, H1, c8(C1))     # re-laid out below if conv1's wgrad is in-place
        self.loss = f32(1)
        # dropout (noisynet.py:456-457, :512-513, :565-566): one keep mask per active site, in the BN input's layout.  The
        # rate is --dropout at every site; --dropout_conv only switches the conv site on (net.NoisyNet does the same)
        self.drop_p = float(a.dropout)
        on = (self.drop_p > 0 and a.dropout_conv > 0, self.drop_p > 0, self.drop_p > 0)
        u8 = lambda *s: torch.zeros(*s, dtype=torch.uint8, device=dev)
        self.keep = [u8(B, C1, P1, P1) if on[0] else None, u8(B, C2, P2, P2) if on[1] else None, u8(B, FC) if on[2] else None]
        self.scratch = torch.zeros(int(self.lib.nn_stage_scratch_bytes(max(C1, C2, FC))) + 64, dtype=torch.uint8, device=dev)
        # weight packs of the step: forward (4 layers) + dgrad (fc2, fc1 as a linear, conv2), one launch
        modes = [NOISE_MERGED if a.merged_dac else NOISE_EXTERNAL, NOISE_EXTERNAL,
                 NOISE_MERGED if a.merged_dac else NOISE_EXTERNAL, NOISE_EXTERNAL]
        self.noise_modes = [m if a.layer_currents[i] > 0 else 0 for i, m in enumerate(modes)]
        W = self._weights()
        shapes = [(C1, 3, fs * fs), (C2, C1, fs * fs), (FC, C2, P2 * P2), (10, FC, 1)]
        self.jobs = (WPrepJob * 7)()
        self.job_layer = [0, 1, 2, 3, 3, 2, 1]
        # (layer, (Cout, Cin, KHW), mode, rows of the consuming GEMM)
        specs = [(0, shapes[0], 0, B * H1 * H1), (1, shapes[1], 0, B * H2 * H2), (2, shapes[2], 0, B), (3, shapes[3], 0, B),
                 (3, shapes[3], 1, B), (2, (FC, C2 * P2 * P2, 1), 1, B), (1, shapes[1], 1, B * P1 * P1)]
        # geometry of the four contractions (fc1 forward / wgrad run as a 5x5 conv over the NHWC pooled map)
        self.geom = [ConvGeom(B, 3, 32, 32, C1, fs, fs, 1, 0), ConvGeom(B, C1, P1, P1, C2, fs, fs, 1, 0),
                     ConvGeom(B, C2, P2, P2, FC, P2, P2, 1, 0), ConvGeom(B, FC, 1, 1, 10, 1, 1, 1, 0)]
        self.geom_fc1_lin = ConvGeom(B, C2 * P2 * P2, 1, 1, FC, 1, 1, 1, 0)
        # conv1 weight gradient through the in-place (shift) kernel: its grad_output lives in the planes layout on the
        # 32x32 input grid, zeroed once here -- nn_stage_bwd only ever writes the 28x28 output positions
        # MaxPool2d and the batch statistics of bn1 fused into the conv1 epilogue (pooled_out + bn_mean): exact, the 104 MB y1n
        # round trip and the pool+statistics pass disappear; the conv1 forward runs on block tiles whose 2x2 windows lie
        # inside one warp.  NN_ENGINE_FUSE_POOL=0: separate stage
        # fc2 + bn4 + loss + their backward as ONE 8-CTA cluster launch (nn_classifier_tail): exact and tested, but it runs
        # ten latency-bound phases on 8 SMs instead of three short launches -- off unless NN_ENGINE_FUSED_TAIL=1
        self.fused_tail = B <= 2048 and self.q_w[3] > 0 and self.q_a[3] > 0 and os.environ.get("NN_ENGINE_FUSED_TAIL", "0") == "1"
        self.fuse_pool1 = bool(self.lib.nn_conv_pool_fusable(C.byref(self.geom[0]), self.noise_modes[0], PREC_BF16)) and \
            os.environ.get("NN_ENGINE_FUSE_POOL", "1") == "1"
        self.bn_scratch = torch.zeros(int(self.lib.nn_conv_bn_scratch_bytes(C1)), dtype=torch.uint8, device=dev)
        # fc1's split-K epilogue also adds the per-channel sums of bn3 (the separate statistics pass is one launch less)
        self.fuse_bn3 = bool(self.lib.nn_conv_linear_bn_fusable(C.byref(self.geom[2]), self.noise_modes[2], PREC_BF16, self.di)) and \
            os.environ.get("NN_ENGINE_FUSE_BN3", "1") == "1"
        self.bn3_scratch = torch.zeros(int(self.lib.nn_stage_scratch_bytes(FC)) + 64, dtype=torch.uint8, device=dev)
        self.gy1_layout = self.lib.nn_conv_wgrad_pack_layout(C.byref(self.geom[0]), PREC_BF16, self.di)
        if self.gy1_layout:
            nbytes = int(self.lib.nn_conv_gy_planes_bytes(C.byref(self.geom[0])))
            self.gyp1 = torch.zeros(nbytes // 16, 8, dtype=torch.bfloat16, device=dev)
        self.wpack = []
        self.wcodes = {}
        for j, (li, (co, ci, khw), mode, m_rows) in enumerate(specs):
            jb = self.jobs[j]
            jb.w_raw = W[li].data_ptr()
            jb.Cout, jb.Cin, jb.KHW, jb.mode, jb.m_rows = co, ci, khw, mode, m_rows
            jb.noise_mode = self.noise_modes[li] if mode == 0 else 0
            jb.want_wsum = 0
            if mode == 0:
                jb.layout = self.lib.nn_conv_pack_layout(C.byref(self.geom[li]), jb.noise_mode, PREC_BF16)
            else:       # dgrad image: the conv layer asks the library, the fc layers run as linear GEMMs (tiled layout)
                jb.layout = self.lib.nn_conv_dgrad_pack_layout(C.byref(self.geom[li]), PREC_BF16) if li == 1 else 0
            jb.q_bits, jb.q_hi = self.q_w[li], 1.0
            if li not in self.wcodes:        # quantizer codes: one scratch per layer, shared by its forward and dgrad jobs
                self.wcodes[li] = torch.zeros(W[li].numel() + 16, dtype=torch.int8, device=dev)
            jb.codes = self.wcodes[li].data_ptr() if self.q_w[li] > 0 else None
            buf = torch.zeros(int(self.lib.nn_weight_pack_bytes(C.byref(jb))) + 1024, dtype=torch.uint8, device=dev)
            jb.packed_out = (buf.data_ptr() + 1023) // 1024 * 1024
            self.wpack.append(buf)
        # conv1 on the shift kernel reads its input as the row-plane image, written by the same launch as xp1 (which the
        # conv1 weight gradient reads)
        self.x1_planes = None
        if self.jobs[0].layout == PACK_SHIFT:
            self.x1_planes = bf16(int(self.lib.nn_conv_shift_planes_bytes(C.byref(self.geom[0]))) // 2)
        self.x1_fwd = self.x1_planes if self.x1_planes is not None else self.xp1
        self.wp_fwd = [self.jobs[i].packed_out for i in range(4)]
        self.wp_dgrad = {3: self.jobs[4].packed_out, 2: self.jobs[5].packed_out, 1: self.jobs[6].packed_out}
        self.wp_dgrad_layout = {3: self.jobs[4].layout, 2: self.jobs[5].layout, 1: self.jobs[6].layout}
        # conv2's dgrad on the resident row-plane kernel: each grad_output image loaded once for all 25 taps (the same
        # NN_PACK_TMA image and bit-identical gx); nn_noisy_conv_dgrad serves geometries it does not
        self.dgrad_planes = self.jobs[6].layout == PACK_TMA and bool(self.lib.nn_conv_dgrad_planes_ok(C.byref(self.geom[1])))
        need = 0
        for g in self.geom + [self.geom_fc1_lin]:
            need = max(need, self.lib.nn_conv_workspace_bytes(C.byref(g), PREC_BF16),
                       self.lib.nn_conv_wgrad_workspace_bytes(C.byref(g), PREC_BF16, self.di))
        self.ws = torch.empty(int(need) + 4096, dtype=torch.uint8, device=dev)
        # the weight gradients run on a side stream next to the dgrad -> stage-backward chain of the same layer (they
        # only share read-only inputs): the small fc kernels and split reduces leave most SMs idle on their own
        self.overlap_wgrad = os.environ.get("NN_ENGINE_OVERLAP_WGRAD", "1") != "0"
        self.side = torch.cuda.Stream(device=dev) if self.overlap_wgrad else None
        self.ws_side = torch.empty(int(need) + 4096, dtype=torch.uint8, device=dev) if self.overlap_wgrad else None
        for p in model.parameters():
            if p.grad is None:
                p.grad = torch.zeros_like(p)
        self._keep_inj = []         # injected keep masks of the step being enqueued
        self.inject = None          # parity hook: dict(u=[...], z=[...], keep=[...]) consumed in the reference's draw order
        self.steps_done = 0         # training steps since the last sync_bn_counters()
        self.logits = f32(B, 10)    # eval_forward output

    def _late_params(self, W):
        early = {id(W[1]), id(W[2]), id(W[3])}
        return [p for _, p in self.opt._params() if id(p) not in early]

    def sync_bn_counters(self):
        """BatchNorm.num_batches_tracked of the four BN modules (state_dict key of the reference model): the kernels keep
        the running statistics, this host-side counter keeps the step count -- call before saving a checkpoint."""
        if self.steps_done:
            for bn in (self.m.bn1, self.m.bn2, self.m.bn3, self.m.bn4):
                if bn.num_batches_tracked is not None:
                    bn.num_batches_tracked += self.steps_done
            self.steps_done = 0

    # ------------------------------------------------------------------ evaluation forward (noisynet.py:1560-1567)
    @torch.no_grad()
    def eval_forward(self, x, currents=None):
        """model.eval() forward of the step's kernels: BatchNorm with running statistics, stochastic rounding off
        (hardware_model.py:283-286), analog noise STILL injected wherever currentN > 0 -- the accurate noise model has no
        training test (hardware_model.py:43); the script switches test noise by mutating args.layer_currents
        (noisynet.py:1551-1553), here: ``currents`` (default: the model's).  Returns the logits [B, 10]."""
        m, a, B, lib, di = self.m, self.a, self.B, self.lib, self.di
        C1, C2, FC, H1, P1, H2, P2 = self.dims
        st = self._st()
        W = self._weights()
        cur_saved = list(a.layer_currents)
        if currents is not None:
            a.layer_currents = list(currents)
        modes_saved = list(self.noise_modes)
        try:
            base = [NOISE_MERGED if a.merged_dac else NOISE_EXTERNAL, NOISE_EXTERNAL,
                    NOISE_MERGED if a.merged_dac else NOISE_EXTERNAL, NOISE_EXTERNAL]
            self.noise_modes = [mo if a.layer_currents[i] > 0 else 0 for i, mo in enumerate(base)]
            if self.noise_modes != modes_saved:
                raise NotImplementedError("eval_forward: the set of noisy layers must match the training configuration "
                                          "(the weight images carry the sigma rows); change the current values only")
            qh1, qh2, qh3, qh4 = (self._qhi(q) for q in (m.quantize1, m.quantize2, m.quantize3, m.quantize4))
            s1, s2, s3, s4 = (_f32(max(h / (2.0 ** b - 1.0), 1e-6)) if b > 0 else 0.0
                              for h, b in ((qh1, a.q_a1), (qh2, a.q_a2), (qh3, a.q_a3), (qh4, a.q_a4)))
            am1, am2, am3 = (float(getattr(a, k, a.act_max)) for k in ("act_max1", "act_max2", "act_max3"))
            self.w_cs = [(_f32(max(2.0 / (2.0 ** b - 1.0), 1e-6)) / 2.0 if b > 0 else 0.0) for b in self.q_w]
            for j in range(4):                                  # forward images only, round-to-nearest weights
                self.jobs[j].stochastic, self.jobs[j].u_inject, self.jobs[j].rng = 0.0, None, Rng(0, 0, None)
            _lib.check(lib.nn_prepare_weights(self.jobs, 4, di, st), "nn_prepare_weights")
            self._input_pack(x, int(a.q_a1), qh1, 0.0, None, Rng(0, 0, None), st)
            self._fwd_gemm(0, self.x1_fwd, s1, self.y1n, self.noise_modes[0], self._absmax(0, W[0]))
            self._stage_fwd(self.y1n, C1, H1, 1, self.pool1, self.amax1, m.bn1, "bn1", a.q_a2, qh2, self.xp2, self.xmax2,
                            act_max=am1, eval_mode=True)
            self._fwd_gemm(1, self.xp2, s2, self.y2n, self.noise_modes[1], self.xmax2)
            self._stage_fwd(self.y2n, C2, H2, 1, self.pool2, self.amax2, m.bn2, "bn2", a.q_a3, qh3, self.xp3, None,
                            act_max=am2, eval_mode=True)
            self._fwd_gemm(2, self.xp3, s3, self.l1n, self.noise_modes[2], self._absmax(2, W[2]))
            self._stage_fwd(self.l1n, FC, 1, 0, None, None, m.bn3, "bn3", a.q_a4, qh4, self.xp4, self.xmax4,
                            act_max=am3, eval_mode=True)
            self._fwd_gemm(3, self.xp4, s4, self.l2n, self.noise_modes[3], self.xmax4)
            bn4 = m.bn4
            _lib.check(lib.nn_head_eval(_p(self.l2n), B, 10, _p(bn4.weight), _p(bn4.bias), _p(bn4.running_mean),
                                        _p(bn4.running_var), float(bn4.eps), _p(self.logits), di, st), "nn_head_eval")
        finally:
            a.layer_currents = cur_saved
            self.noise_modes = modes_saved
        return self.logits

    # ------------------------------------------------------------------ helpers
    def _weights(self):
        m = self.m
        return [m.conv1.weight, m.conv2.weight, m.linear1.weight, m.linear2.weight]

    def _rng(self):
        return ops.next_rng(self.di)

    def _st(self):
        return torch.cuda.current_stream(self.di).cuda_stream

    def _take(self, kind):
        if self.inject is None or not self.inject.get(kind):
            return None
        return self.inject[kind].pop(0)

    def _absmax(self, idx, w):
        hit = self.m.w_absmax.get(idx)
        if hit is not None and hit[0] == w._version:
            return hit[1]
        return ops.tensor_stats(w.detach())[1:2]

    def _input_pack(self, x, q_bits, q_hi, stoch, u, rng, stream, gathered=False):
        """conv1's input codes: the NHWC image xp1 and, for the shift kernel, the row-plane image from the same pass (from
        xp1 when ``gathered``: nn_input_gather_quant_pack has written it)"""
        lib, B = self.lib, self.B
        if self.x1_planes is None:
            if not gathered:
                _lib.check(lib.nn_input_quant_pack(_p(x), _p(self.xp1), None, B, 3, 32 * 32, 8, q_bits, q_hi, stoch, _p(u), rng,
                                                   self.di, stream), "nn_input_quant_pack")
            return
        g = self.geom[0]
        _lib.check(lib.nn_input_quant_pack_rows(None if gathered else _p(x), _p(self.xp1), _p(self.x1_planes), B, 3, 32, 32, g.KW,
                                                q_bits, q_hi, stoch, _p(u), rng, self.di, stream), "nn_input_quant_pack_rows")

    def _fwd_gemm(self, idx, xp, a_cs, y_noisy, mode, scale_dev, z=None, pooled=None, argmax=None, bn=None, key=None, zero=None,
                  eval_mode=False):
        a = ConvFwdArgs()
        a.g = self.geom[idx]
        a.x = None
        a.x_packed = _p(xp)
        a.w_eff, a.w_raw, a.w_packed = None, None, self.wp_fwd[idx]
        a.w_packed_layout = self.jobs[idx].layout
        cur = float(self.a.layer_currents[idx])
        if cur > 0:
            a.y, a.y_noisy = None, _p(y_noisy)
            a.noise_mode, a.current = mode, cur
            a.scale_dev = _p(scale_dev)
            a.z_inject = _p(z)
            a.rng = Rng(0, 0, None) if z is not None else self._rng()
        else:                                   # currentN == 0: no analog noise on this layer (noisynet.py:414)
            a.y, a.y_noisy, a.noise_mode = _p(y_noisy), None, 0
        if pooled is not None:                  # MaxPool2d(2,2) fused into the conv epilogue: the full-size output is never written
            a.y, a.y_noisy = None, None
            a.pooled_out, a.argmax_out = _p(pooled), _p(argmax)
        if bn is not None:                      # the BatchNorm statistics of the (pooled) output come from the same launch
            a.bn_mean, a.bn_invstd = _p(self.stat[key][0]), _p(self.stat[key][1])
            a.bn_running_mean, a.bn_running_var = _p(bn.running_mean), _p(bn.running_var)
            a.bn_eps, a.bn_momentum, a.bn_eval_mode = float(bn.eps), float(bn.momentum), 1 if eval_mode else 0
            a.bn_scratch, a.zero_out = _p(self.bn_scratch if pooled is not None else self.bn3_scratch), _p(zero)
        a.precision = PREC_BF16
        a.a_code_scale, a.w_code_scale = a_cs, self.w_cs[idx]
        a.workspace, a.workspace_bytes = _p(self.ws), self.ws.numel()
        _lib.check(self.lib.nn_noisy_conv_fwd(C.byref(a), self.di, self._st()), "nn_noisy_conv_fwd")

    def _wgrad(self, idx, gyp, xp, a_cs, w_raw, gw, gy_layout=0):
        if self.side is None:
            return self._wgrad_on(self.ws, idx, gyp, xp, a_cs, w_raw, gw, gy_layout)
        self.side.wait_stream(torch.cuda.current_stream(self.di))       # grad_output / activations of this layer are ready
        with torch.cuda.stream(self.side):
            self._wgrad_on(self.ws_side, idx, gyp, xp, a_cs, w_raw, gw, gy_layout)

    def _wgrad_on(self, ws, idx, gyp, xp, a_cs, w_raw, gw, gy_layout=0):
        a = ConvWgradArgs()
        a.g = self.geom[idx]
        a.gy, a.x, a.gw = None, None, _p(gw)
        a.gy_packed, a.x_packed, a.gy_packed_layout = _p(gyp), _p(xp), gy_layout
        if self.q_w[idx] > 0:
            a.w_raw, a.w_lo, a.w_hi = _p(w_raw), -1.0, 1.0        # STE of the weight quantizer (hardware_model.py:323)
        a.precision, a.a_code_scale = PREC_BF16, a_cs
        a.workspace, a.workspace_bytes = _p(ws), ws.numel()
        _lib.check(self.lib.nn_noisy_conv_wgrad(C.byref(a), self.di, self._st()), "nn_noisy_conv_wgrad")

    def _dgrad(self, geom, gyp, layer, gx):
        a = ConvDgradArgs()
        a.g = geom
        a.gy, a.gy_packed, a.w_eff, a.w_packed, a.gx = None, _p(gyp), None, self.wp_dgrad[layer], _p(gx)
        a.w_packed_layout = self.wp_dgrad_layout[layer]
        a.precision, a.w_code_scale = PREC_BF16, self.w_cs[layer]
        a.workspace, a.workspace_bytes = _p(self.ws), self.ws.numel()
        if layer == 1 and self.dgrad_planes:
            _lib.check(self.lib.nn_conv_dgrad_planes(C.byref(a), self.di, self._st()), "nn_conv_dgrad_planes")
        else:
            _lib.check(self.lib.nn_noisy_conv_dgrad(C.byref(a), self.di, self._st()), "nn_noisy_conv_dgrad")

    def _stage_fwd(self, x_in, C_, H, pool, pooled, amax, bn, key, q_bits, q_hi, xp, xmax, u=None, act_max=None, eval_mode=False,
                   stats_ready=False, site=None):
        a = StageArgs()
        a.eval_mode = 1 if eval_mode else 0
        a.stats_ready = 1 if stats_ready else 0
        a.in_ = _p(x_in)
        a.B, a.C, a.H, a.W, a.pool = self.B, C_, H, H, pool
        a.pooled, a.argmax = _p(pooled), _p(amax)
        a.gamma, a.beta = _p(bn.weight), _p(bn.bias)
        a.running_mean, a.running_var = _p(bn.running_mean), _p(bn.running_var)
        a.momentum, a.eps = float(bn.momentum), float(bn.eps)
        a.mean, a.invstd = _p(self.stat[key][0]), _p(self.stat[key][1])
        a.act_max = float(self.a.act_max if act_max is None else act_max)
        a.q_bits, a.q_hi = int(q_bits), float(q_hi)
        a.stochastic = float(self.a.stochastic) if (self.m.training and not eval_mode) else 0.0
        a.u_inject = _p(u)
        a.rng = Rng(0, 0, None) if u is not None else self._rng()
        a.xp, a.Cp = _p(xp), xp.shape[-1]
        a.act, a.xmax_out = None, _p(xmax)
        a.scratch = _p(self.scratch)
        keep = self.keep[site] if site is not None else None
        if keep is not None and not eval_mode:             # dropout is the identity in eval
            a.drop_p, a.keep = self.drop_p, _p(keep)
            ki = self._take("keep")
            self._keep_inj.append(ki)                      # alive until the launch has run
            a.keep_inject = _p(ki)
            a.drop_rng = Rng(0, 0, None) if ki is not None else self._rng()     # drawn only when p > 0
        _lib.check(self.lib.nn_stage_fwd(C.byref(a), self.di, self._st()), "nn_stage_fwd")

    def _stage_bwd(self, g, x, amax, C_, H, pool, bn, key, q_bits, q_hi, gyp, planes_grid=None, act_max=None, site=None):
        a = StageBwdArgs()
        a.g, a.x, a.argmax = _p(g), _p(x), _p(amax)
        a.B, a.C, a.H, a.W, a.pool = self.B, C_, H, H, pool
        a.mean, a.invstd = _p(self.stat[key][0]), _p(self.stat[key][1])
        a.gamma, a.beta = _p(bn.weight), _p(bn.bias)
        a.act_max, a.q_bits, a.q_hi = float(self.a.act_max if act_max is None else act_max), int(q_bits), float(q_hi)
        a.dgamma, a.dbeta = _p(bn.weight.grad), _p(bn.bias.grad)
        a.gyp, a.Cp, a.gy_f32 = _p(gyp), (C_ + 7) // 8 * 8, None
        if planes_grid is not None:
            a.gy_layout, a.virt_H, a.virt_W = PACK_SHIFT, planes_grid[0], planes_grid[1]
        a.scratch = _p(self.scratch)
        keep = self.keep[site] if site is not None else None
        if keep is not None:
            a.drop_p, a.keep = self.drop_p, _p(keep)
        _lib.check(self.lib.nn_stage_bwd(C.byref(a), self.di, self._st()), "nn_stage_bwd")

    def _qhi(self, qm):
        """Fixed quantisation range of a QuantMeasure (hardware_model.py:265-271, host values cached)."""
        if qm.num_bits <= 0:
            return 0.0
        if qm.max_value > 0:
            return float(qm.max_value)
        v = qm._host('running_max')
        if v <= 0:
            raise RuntimeError("NoisyNetEngine needs calibrated activation ranges (running_max > 0)")
        return v

    # ------------------------------------------------------------------ one training step
    @torch.no_grad()
    def train_step(self, x, labels, gather=None):
        """One training step.  ``x`` [B,3,32,32] fp32 + ``labels`` [B] int64 on the device; or, with
        ``gather=(idx, aug)``, ``x`` is the whole resident zero-padded dataset [N,3,Hp,Wp] (utils.py:165-167), ``idx`` [B]
        int64 the batch's sample indices and ``aug`` a device int32[3] {off_y, off_x, flip} (noisynet.py:1261-1269):
        the batch is assembled inside the input-quantizer kernel; ``labels`` are then the batch's labels."""
        m, a, B, lib, di = self.m, self.a, self.B, self.lib, self.di
        C1, C2, FC, H1, P1, H2, P2 = self.dims
        st = self._st()
        W = self._weights()
        stoch = float(a.stochastic) if m.training else 0.0
        am1, am2, am3 = (float(getattr(a, k, a.act_max)) for k in ("act_max1", "act_max2", "act_max3"))   # noisynet.py:887-889
        self.steps_done += 1
        qh1, qh2, qh3, qh4 = (self._qhi(q) for q in (m.quantize1, m.quantize2, m.quantize3, m.quantize4))
        s1, s2, s3, s4 = (_f32(max(h / (2.0 ** b - 1.0), 1e-6)) if b > 0 else 0.0
                          for h, b in ((qh1, a.q_a1), (qh2, a.q_a2), (qh3, a.q_a3), (qh4, a.q_a4)))
        self.w_cs = [(_f32(max(2.0 / (2.0 ** b - 1.0), 1e-6)) / 2.0 if b > 0 else 0.0) for b in self.q_w]
        # ---- weights: quantize (stochastic rounding) + pack for forward and dgrad, all layers, ONE launch
        self._uw_keep = []
        self._keep_inj = []
        for li in range(4):
            uw = self._take("uw")
            self._uw_keep.append(uw)             # keep injected tensors alive until the launch below has run
            rng = Rng(0, 0, None) if uw is not None else self._rng()
            for j in range(7):
                if self.job_layer[j] == li:
                    self.jobs[j].stochastic = stoch
                    self.jobs[j].u_inject = _p(uw)
                    self.jobs[j].rng = rng
        u = self._take("u")
        rng_in = Rng(0, 0, None) if u is not None else self._rng()

        def input_pack(stream):
            if gather is not None:
                idx, aug = gather
                _lib.check(lib.nn_input_gather_quant_pack(_p(x), _p(idx), B, 3, x.shape[2], x.shape[3], 32, 32, 0, 0, 0, _p(aug),
                                                          _p(self.xp1), None, 8, int(a.q_a1), qh1, stoch, _p(u), rng_in, di, stream),
                           "nn_input_gather_quant_pack")
                self._input_pack(None, int(a.q_a1), qh1, stoch, None, Rng(0, 0, None), stream, gathered=True)
            else:
                self._input_pack(x, int(a.q_a1), qh1, stoch, u, rng_in, stream)

        if self.side is not None:
            # conv1's image is needed at once; the other six (fc1 is 90 % of the bytes) are packed on the side stream
            # while the input pack and the conv1 forward run, and joined before conv2.  (Moving the input pack to the side
            # stream as well, next to conv1's image, would delay the six images.)
            self.side.wait_stream(torch.cuda.current_stream(di))
            with torch.cuda.stream(self.side):
                _lib.check(lib.nn_prepare_weights(C.byref(self.jobs[1]), 6, di, self._st()), "nn_prepare_weights")
            _lib.check(lib.nn_prepare_weights(self.jobs, 1, di, st), "nn_prepare_weights")
        else:
            _lib.check(lib.nn_prepare_weights(self.jobs, 7, di, st), "nn_prepare_weights")
        input_pack(st)
        # ---- forward
        if self.fuse_pool1:
            # conv1 + analog noise + MaxPool2d + the batch statistics of bn1 in ONE launch: the 104 MB fp32 conv output is
            # never written; the stage that follows only normalises, quantizes and packs
            self._fwd_gemm(0, self.x1_fwd, s1, None, self.noise_modes[0], self._absmax(0, W[0]), self._take("z"),
                           pooled=self.pool1, argmax=self.amax1, bn=m.bn1, key="bn1", zero=self.xmax2)
            self._stage_fwd(self.pool1, C1, P1, 0, None, None, m.bn1, "bn1", a.q_a2, qh2, self.xp2, self.xmax2, self._take("u"), act_max=am1,
                            stats_ready=True, site=0)
        else:
            self._fwd_gemm(0, self.x1_fwd, s1, self.y1n, self.noise_modes[0], self._absmax(0, W[0]), self._take("z"))
            self._stage_fwd(self.y1n, C1, H1, 1, self.pool1, self.amax1, m.bn1, "bn1", a.q_a2, qh2, self.xp2, self.xmax2, self._take("u"), act_max=am1,
                            site=0)
        if self.side is not None:
            torch.cuda.current_stream(di).wait_stream(self.side)
        self._fwd_gemm(1, self.xp2, s2, self.y2n, self.noise_modes[1], self.xmax2, self._take("z"))
        self._stage_fwd(self.y2n, C2, H2, 1, self.pool2, self.amax2, m.bn2, "bn2", a.q_a3, qh3, self.xp3, None, self._take("u"), act_max=am2,
                        site=1)
        z3 = self._take("z")
        if self.fuse_bn3 and z3 is None:        # (injected draws run the general epilogue, which is not split over K)
            self._fwd_gemm(2, self.xp3, s3, self.l1n, self.noise_modes[2], self._absmax(2, W[2]), None, bn=m.bn3, key="bn3", zero=self.xmax4)
            self._stage_fwd(self.l1n, FC, 1, 0, None, None, m.bn3, "bn3", a.q_a4, qh4, self.xp4, self.xmax4, self._take("u"), act_max=am3,
                            stats_ready=True, site=2)
        else:
            self._fwd_gemm(2, self.xp3, s3, self.l1n, self.noise_modes[2], self._absmax(2, W[2]), z3)
            self._stage_fwd(self.l1n, FC, 1, 0, None, None, m.bn3, "bn3", a.q_a4, qh4, self.xp4, self.xmax4, self._take("u"), act_max=am3,
                            site=2)
        bn4 = m.bn4
        if self.fused_tail:
            # fc2 forward + noise, bn4, cross entropy, their backward and the fc2 dgrad: one 8-CTA cluster launch
            t = TailArgs()
            t.xp, t.B, t.K, t.Kp, t.C = _p(self.xp4), B, FC, self.xp4.shape[-1], 10
            t.w_codes, t.w_raw = self.wcodes[3].data_ptr(), _p(W[3])
            t.a_code_scale, t.w_code_scale = s4, self.w_cs[3]
            cur = float(a.layer_currents[3])
            z = self._take("z")
            if cur > 0:
                t.noise_mode, t.current, t.scale_dev, t.z_inject = self.noise_modes[3], cur, _p(self.xmax4), _p(z)
                t.rng = Rng(0, 0, None) if z is not None else self._rng()
            t.labels, t.gamma, t.beta = _p(labels), _p(bn4.weight), _p(bn4.bias)
            t.running_mean, t.running_var = _p(bn4.running_mean), _p(bn4.running_var)
            t.momentum, t.eps = float(bn4.momentum), float(bn4.eps)
            t.loss_out, t.logits_out, t.g, t.g_packed, t.Cp_g = _p(self.loss), _p(self.l2n), _p(self.g4), _p(self.gyp4), 16
            t.gx, t.dgamma, t.dbeta = _p(self.gx4), _p(bn4.weight.grad), _p(bn4.bias.grad)
            _lib.check(lib.nn_classifier_tail(C.byref(t), di, st), "nn_classifier_tail")
            self._wgrad(3, self.gyp4, self.xp4, s4, W[3], W[3].grad)
        else:
            self._fwd_gemm(3, self.xp4, s4, self.l2n, self.noise_modes[3], self.xmax4, self._take("z"))
            _lib.check(lib.nn_head_fwd_bwd(_p(self.l2n), _p(labels), B, 10, _p(bn4.weight), _p(bn4.bias), _p(bn4.running_mean),
                                           _p(bn4.running_var), float(bn4.momentum), float(bn4.eps), _p(self.loss), None,
                                           _p(self.g4), _p(self.gyp4), 16, _p(bn4.weight.grad), _p(bn4.bias.grad), di, st),
                       "nn_head_fwd_bwd")
            # ---- backward
            self._wgrad(3, self.gyp4, self.xp4, s4, W[3], W[3].grad)
            self._dgrad(self.geom[3], self.gyp4, 3, self.gx4)
        self._stage_bwd(self.gx4, self.l1n, None, FC, 1, 0, m.bn3, "bn3", a.q_a4, qh4, self.gyp3, act_max=am3, site=2)
        self._wgrad(2, self.gyp3, self.xp3, s3, W[2], W[2].grad)
        if self.red is not None:        # fc gradients (85 % of the payload) travel while the conv backward runs
            if self.side is not None:
                with torch.cuda.stream(self.side):
                    self.red.start_early()
            else:
                self.red.start_early()
        self._dgrad(self.geom_fc1_lin, self.gyp3, 2, self.gx3)
        self._stage_bwd(self.gx3, self.pool2, self.amax2, C2, H2, 1, m.bn2, "bn2", a.q_a3, qh3, self.gyp2, act_max=am2, site=1)
        self._wgrad(1, self.gyp2, self.xp2, s2, W[1], W[1].grad)
        if self.red is not None:        # second early bucket: conv2's weight gradient
            if self.side is not None:
                with torch.cuda.stream(self.side):
                    self.red.start_early(1)
            else:
                self.red.start_early(1)
        early_update = self.opt is not None and self.side is not None and hasattr(self.opt, "step_part")
        if early_update:
            # fc2, fc1 and conv2 (99.8 % of the parameters): gradients final (and exchanged) -> AdamW + clamp + max|W| now, on
            # the side stream under conv2's dgrad and the stage-1 backward; only conv1 and the BatchNorm vectors wait for
            # the end of the step.  Nothing left on the main stream reads these weights (dgrad uses the packed images).
            with torch.cuda.stream(self.side):
                if self.red is not None:
                    self.red.wait_early(0)
                    self.red.wait_early(1)
                self.opt.step_part([W[3], W[2], W[1]], advance=False)
        self._dgrad(self.geom[1], self.gyp2, 1, self.gx2)
        self._stage_bwd(self.gx2, self.pool1, self.amax1, C1, H1, 1, m.bn1, "bn1", a.q_a2, qh2, self.gyp1,
                        planes_grid=(32, 32) if self.gy1_layout else None, act_max=am1, site=0)
        self._wgrad(0, self.gyp1, self.xp1, s1, W[0], W[0].grad, self.gy1_layout)
        # ---- exchange + update
        if self.side is not None:
            torch.cuda.current_stream(di).wait_stream(self.side)
        if self.red is not None:
            self.red.all_reduce_sum_()
        if self.opt is not None:
            if early_update:
                self.opt.step_part(self._late_params(W), advance=True)
            else:
                self.opt.step()
            for idx, w in enumerate(W):
                m.w_absmax[idx] = (w._version, self.opt.absmax_of(w))
        return self.loss
