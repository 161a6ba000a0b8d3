"""The launch shadow (test infrastructure): every `ops` wrapper a reference in tests/launch_refs.py covers is replaced
by one that runs the real kernel and compares its outputs with the reference computed from the inputs the kernel
actually received (pre-call copies of the operands the call overwrites and also reads); every other public `ops`
function is counted, and a scenario that calls one which is neither checked nor listed in UNCHECKED fails.  Used by
tests/test_step_launches_gpu.py (the benchmarked steps) and tests/test_path_launches_gpu.py (the sampling variants, the
VAE encoder and the annotators).  `pytest -s` prints one line per distinct call signature with its plan and errors.
"""
import collections
import gc
import inspect
import math
import os
import sys
import traceback

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import launch_refs as R  # noqa: E402
from tolerances import close  # noqa: E402

# op -> (max-abs bound as a fraction of max|ref|, norm-relative bound): the bounds of each op's per-kernel test
BOUNDS = {
    "gemm": (2e-3, 1e-3),             # test_gemm_*_gpu.py
    "groupnorm": (3e-3, 1e-3),        # test_kernels_gpu.py
    "layernorm": (3e-3, 1e-3),
    "attention": (3e-3, 1e-3),        # test_kernels_gpu.py / test_attention_fwd_gpu.py
    "wgrad_tn": (1e-3, 1e-3),         # test_train_kernels_gpu.py
    "attention_bwd": (5e-3, 1e-3),
    "groupnorm_bwd": (4e-3, 1e-3),
    "layernorm_bwd": (4e-3, 1e-3),
    "gemm_relu": (2e-3, 1e-3),        # gemm's: test_hed_gpu.py holds it bit-equal to gemm(...).clamp_min(0)
    "softmax_rows": (2e-3, 1e-3),     # test_round2_kernels_gpu.py
    "weighted_sum": (2e-3, 1e-3),
    "gaussian_sample": (1e-5, 1e-6),
    # the norm-relative bounds of test_lineart_gpu.py (NORM_BOUND, OUT_BOUND) and test_hed_gpu.py (SIDE_KERNEL_BOUND).
    # Those tests hold no max-abs bound, so these guards were measured on an H100 80GB HBM3 at 700 W over the
    # scenarios of test_path_launches_gpu.py, as a fraction of max|ref|: instance_norm up to 4.22e-4 (the fp16 rounding
    # of the output alone may reach 2^-11 = 4.9e-4 of it, hence 6e-4); lineart_out up to 9.28e-7 (fp32 sums of 3136
    # products in another order); hed_side_pool up to 3.50e-7
    "instance_norm": (6e-4, 4e-4),
    "lineart_out": (1.2e-6, 1e-6),
    "hed_side_pool": (4.5e-7, 1e-6),
}
# ops compared bit for bit: gathers, a nearest-neighbour copy and a max
EXACT = ("tap_gather", "im2col_s2", "upsample2x", "max_pool2x2")
# A finding: attention_bwd's dq and dk of the steps' self-attention calls exceed the 1e-3 bound their per-kernel test
# holds on random operands.  Measured on an H100 per image, norm-relative: dq up to 2.26e-3 against autograd (pretrain
# step, 1024 x 1024 keys, d 80), dk up to 1.6e-3 (4096 x 4096, d 40); dv, which does not involve the softmax gradient,
# stays at 4e-4.  Most of it is the forward's fp16 output o, from which the kernel forms the row term rowsum(dout * o):
# its rounding enters every dS = P (dP - rowsum) of a row whose P is close to uniform -- self-attention over smooth
# activations -- and cancels there.  Against the same formula with the o the kernel received
# (launch_refs.attention_dqk_given_o) dq and dk stay below 1e-3 except at 4096 keys, d 40: up to 1.38e-3, the kernel's
# own fp16 products summed over 4096 keys.  The bounds are set about 20 % above these figures.
ATTN_DQK = (5e-3, 2.7e-3)
ATTN_DQK_GIVEN_O = (5e-3, 1.7e-3)
GN_STATS = (2e-3, 1e-4)               # {sum, sumsq} against fp64 sums (test_round2_kernels_gpu.py)
LSE_ABS = 2e-3                        # |lse - ref| <= 2e-3 * max(1, max|ref|) (log2 domain)

# ops functions the scenarios call that the shadow does not check, and why
UNCHECKED = {
    "zeros": "cudaMemsetAsync of a new buffer, no kernel (test_round2_kernels_gpu.py)",
    "small_linear": "time-embedding MLP and emb_layers GEMV, fp32 against torch in test_kernels_gpu.py / "
                    "test_round2_kernels_gpu.py at the steps' row counts",
    "timestep_embedding": "bit-exact against the reference formula in test_kernels_gpu.py",
    "cast_transpose": "weight preparation, bit-exact cast in test_kernels_gpu.py",
    "nchw_to_nhwc_f16": "layout conversion, bit-exact in test_kernels_gpu.py",
    "nhwc_to_nchw_f32": "layout conversion, bit-exact in test_kernels_gpu.py",
    "im2col_3x3": "gather of the dense conv weight gradients, bit-exact in test_round2_kernels_gpu.py",
    "q_sample": "bit-exact in test_round2_kernels_gpu.py",
    "mse_loss_grad": "loss and its gradient, test_train_kernels_gpu.py at the trainer's loss scale",
    "geglu_fwd": "test_train_kernels_gpu.py at the feed-forward widths",
    "geglu_bwd": "test_train_kernels_gpu.py at the feed-forward widths",
    "colsum": "bias gradients, test_round2_kernels_gpu.py / test_train_kernels_gpu.py",
    "image_colsum": "per-image time-embedding gradients, test_train_kernels_gpu.py",
    "outer_accum": "emb_layers weight gradients, test_round2_kernels_gpu.py",
    "silu_bwd": "test_round2_kernels_gpu.py",
    "copy2d": "strided fp32 copies of gradient slices, test_round2_kernels_gpu.py",
    "upsample2x_bwd": "test_train_kernels_gpu.py",
    "im2col_s2_bwd": "test_train_kernels_gpu.py",
    "transpose_f16": "transposed weight copies for the data gradients, bit-exact in test_round2_kernels_gpu.py",
    "conv_dgrad_weight": "data-gradient weight copies, bit-exact in test_round2_kernels_gpu.py",
    "cast_rows": "fp32 -> fp16 row cast, test_conditioning_kernels_gpu.py",
    "nonfinite_flag": "overflow flag of the loss scaling, test_round2_kernels_gpu.py",
    "hed_fuse": "float64 post-process of the side maps, against cv2 / numpy on the network's own maps in "
                "test_hed_gpu.py",
    "openpose_resample": "float64 post-process, against cv2 on the network's own maps in test_openpose_gpu.py",
    "openpose_smooth": "float64 post-process, against scipy.ndimage in test_openpose_gpu.py",
    "openpose_peaks": "float64 post-process, against numpy in test_openpose_gpu.py",
    "openpose_limbs": "float64 post-process, against the numpy restatement in test_openpose_gpu.py",
}

COVERED = tuple(BOUNDS) + EXACT


# ------------------------------------------------------------------------------------------------------ the shadow
def _span(t):
    lo = t.data_ptr()
    return lo, lo + (sum((n - 1) * s for n, s in zip(t.shape, t.stride())) + 1) * t.element_size()


def _overlaps(t, outs):
    if t is None or t.numel() == 0:
        return False
    lo, hi = _span(t)
    return any(o is not None and o.numel() and lo < _span(o)[1] and _span(o)[0] < hi for o in outs)


def _tensors(v):
    if torch.is_tensor(v):
        return [v]
    if isinstance(v, dict):
        return [t for t in v.values() if torch.is_tensor(t)]
    if isinstance(v, (list, tuple)):
        return [t for t in v if torch.is_tensor(t)]
    return []


# op -> (argument names the call reads, argument names it writes)
IO = {
    "gemm": (("a", "w", "a2", "w2", "bias", "rowbias", "residual", "hi"), ("out", "seg_outs", "dup_out")),
    "groupnorm": (("x1", "add1", "x2", "add2", "gamma", "beta", "gamma_hi", "beta_hi"), ("out",)),
    "layernorm": (("x", "gamma", "beta", "gamma_hi", "beta_hi"), ()),
    "attention": (("q", "k", "vt"), ("out", "lse")),
    "wgrad_tn": (("a", "b", "out"), ("out",)),
    "attention_bwd": (("q", "k", "v", "o", "dout", "lse"), ("dq", "dk", "dv")),
    "groupnorm_bwd": (("dy", "fwd_stats", "x1", "add1", "x2", "add2", "gamma", "beta", "dgamma", "dbeta", "res"),
                      ("dgamma", "dbeta")),
    "layernorm_bwd": (("x", "dy", "gamma", "dgamma", "dbeta", "res"), ("dgamma", "dbeta")),
    "im2col_s2": (("x",), ()),
    "upsample2x": (("x",), ()),
    "softmax_rows": (("logits",), ()),
    "weighted_sum": (("tensors",), ("out",)),
    "gaussian_sample": (("moments", "noise"), ()),
    "tap_gather": (("x",), ("out",)),
    "instance_norm": (("x", "residual"), ("out",)),
    "lineart_out": (("x", "weight", "bias"), ()),
    "hed_side_pool": (("x", "weight", "bias"), ()),
    "max_pool2x2": (("x",), ()),
}
IO["gemm_relu"] = IO["gemm"]


def _clone_read_and_written(name, p):
    """copies of the operands the call reads and (possibly through an alias) overwrites"""
    reads, writes = IO[name]
    outs = [t for w in writes for t in _tensors(p.get(w))]
    sub = dict(p)
    for r in reads:
        v = p.get(r)
        if isinstance(v, dict):
            sub[r] = {k: (t.clone() if torch.is_tensor(t) and _overlaps(t, outs) else t) for k, t in v.items()}
        elif isinstance(v, (list, tuple)):
            sub[r] = [t.clone() if torch.is_tensor(t) and _overlaps(t, outs) else t for t in v]
        elif torch.is_tensor(v) and _overlaps(v, outs):
            sub[r] = v.clone()
    aliased = sorted(r for r in reads if any(_overlaps(t, outs) for t in _tensors(p.get(r))))
    return sub, aliased


def _halves(t):
    h = t.shape[0] // 2
    return [("lo", t[:h]), ("hi", t[h:])]


def _tma_ok(t, ld):
    return t.data_ptr() % 16 == 0 and ld % 8 == 0


def _gemm_epilogue(p):
    """'tma' when the arguments let ctrlora_gemm_f16 store through the TMA epilogue (gemm_sm90.cu, tma_epi), else
    'rpt' (row per thread).  Split tiles use the row-per-thread epilogue either way."""
    if p["out_f32"]:
        return "rpt"
    res = p["residual"]
    if res is not None and (res.dtype == torch.float32 or not _tma_ok(res, res.stride(-2))):
        return "rpt"
    if p["seg_outs"] is None:
        if p["out"] is None:  # allocated by the wrapper: aligned, row stride N
            return "tma" if (p["w"].shape[0] // (2 if p["geglu"] else 1)) % 8 == 0 else "rpt"
        return "tma" if _tma_ok(p["out"], p["out"].stride(-2)) else "rpt"
    segs = [o for o, t in zip(p["seg_outs"], p["transposed"]) if not t]
    if not segs or p["transposed"][0]:
        return "rpt"
    return "tma" if all(_tma_ok(o, p["seg_width"]) for o in segs) else "rpt"


def _fmt_shape(t):
    return "x".join(map(str, t.shape)) if torch.is_tensor(t) else "-"


def _describe(name, p):
    """(shape text, plan text) of one call for the report"""
    if name in ("gemm", "gemm_relu"):
        a, w = p["a"], p["w"]
        m = a.shape[0] if a.dim() == 2 else a.shape[0] * a.shape[1] * a.shape[2]
        flags = [f for f, on in (("hi", p["hi"] is not None), ("geglu", p["geglu"]), ("a2", p["a2"] is not None),
                                 ("res", p["residual"] is not None), ("rowbias", p["rowbias"] is not None),
                                 ("f32", p["out_f32"]), ("scale", p["out_scale"] != 1.0),
                                 ("segs" + "".join(str(int(t)) for t in p["transposed"][:len(p["seg_outs"] or [])]),
                                  p["seg_outs"] is not None), ("dup", p["dup_out"] is not None)) if on]
        shape = f"{_fmt_shape(a)} M={m} K={p['ksize'] ** 2}x{a.shape[-1]} N={w.shape[0]} " + ",".join(flags)
        plan = f"bn={p['block_n'] or 'auto'} epi={_gemm_epilogue(p)}"
    elif name == "wgrad_tn":
        shape = f"M={p['a'].shape[0]} P={p['a'].shape[1]} Q={p['b'].shape[1]} beta={p['beta']:g}"
        plan = ""
    elif name in ("groupnorm", "groupnorm_bwd"):
        x1, x2 = p["x1"], p["x2"]
        shape = f"{_fmt_shape(x1)}" + (f"+{x2.shape[-1]}" if x2 is not None else "") + \
            "".join(f",{k}" for k in ("add1", "add2", "gamma_hi", "res", "dgamma") if p.get(k) is not None) + \
            (",silu" if p["silu"] else "")
        plan = ""
    elif name in ("attention", "attention_bwd"):
        shape = f"B={p['batch']} H={p['heads']} nq={p['nq']} nk={p['nk']} d={p['head_dim']}"
        plan = ""
    elif name == "tap_gather":
        x = p["x"]
        shape = f"{_fmt_shape(x)} {'f32nchw' if x.dtype == torch.float32 else 'f16'}" + \
            (f" C={p['channels']}" if p["channels"] else "") + \
            f" taps={len(p['taps'])} {'reflect' if p['reflect'] else 'zero'} k_pad={p['k_pad']}"
        plan = ""
    elif name == "softmax_rows":
        shape, plan = f"{_fmt_shape(p['logits'])} scale={p['scale']:.4g}", ""
    elif name == "weighted_sum":
        shape = f"{len(p['tensors'])}x{_fmt_shape(p['tensors'][0])} w=" + ",".join(f"{w:g}" for w in p["weights"])
        plan = ""
    elif name == "gaussian_sample":
        shape = _fmt_shape(p["moments"]) + (",noise" if p["noise"] is not None else "") + f" scale={p['scale']:g}"
        plan = ""
    else:
        flags = [k for k in ("phases", "relu", "residual", "want_u8", "pool")
                 if p.get(k) is not None and p[k] is not False]
        shape = _fmt_shape(p["x"]) + (",hi" if p.get("gamma_hi") is not None else "") + \
            (",res" if p.get("res") is not None else "") + (f" pad_lo={p['pad_lo']}" if name == "im2col_s2" else "") + \
            "".join(f",{k}" for k in flags)
        plan = ""
    return shape, plan


def _call_site():
    """file:line of the innermost frame outside ops.py and this test machinery"""
    skip = (os.path.join("ctrlora_b200", "ops.py"), "launch_refs.py", os.path.basename(__file__))
    for fr in reversed(traceback.extract_stack()[:-1]):
        if not fr.filename.endswith(skip):
            return f"{os.path.relpath(fr.filename, ROOT)}:{fr.lineno}"
    return "?"


class Shadow:
    """Replaces the covered `ops` wrappers by checked ones and every other public `ops` function by a counted one.
    Calls made from inside a wrapper (ops.gemm's two-launch fallback calls ops.gemm) run unchecked: the outer call is
    checked as a whole."""

    def __init__(self, monkeypatch, replace=None, only=COVERED):
        from ctrlora_b200 import ops
        self.ops = ops
        self.only = only
        self.grouped = collections.defaultdict(set)  # op -> batch sizes of its grouped (two-network) calls
        self.calls = collections.Counter()
        self.records = collections.OrderedDict()   # (op, shape, plan) -> [count, worst error, call site]
        self.failures = []                          # (op, call site, shape, message)
        self.split_calls = 0
        self._depth = 0
        self._abs = 0.0
        replace = replace or {}
        members = inspect.getmembers(ops, inspect.isfunction)
        for name, fn in members:
            if fn.__module__ != ops.__name__ or name.startswith("_"):
                continue
            real = replace.get(name, fn)
            monkeypatch.setattr(ops, name, self._wrap(name, real, _signature(dict(members), name)))

    def _wrap(self, name, real, sig):
        def wrapper(*args, **kwargs):
            if self._depth:
                return real(*args, **kwargs)
            self.calls[name] += 1
            self._depth += 1
            try:
                if name not in self.only:
                    return real(*args, **kwargs)
                return self._checked(name, real, sig, args, kwargs)
            finally:
                self._depth -= 1
        return wrapper

    def _checked(self, name, real, sig, args, kwargs):
        bound = sig.bind(*args, **kwargs)
        bound.apply_defaults()
        p = dict(bound.arguments)
        sub, aliased = _clone_read_and_written(name, p)
        if p.get("hi") is not None or p.get("gamma_hi") is not None:
            lead = p["a"] if name in ("gemm", "gemm_relu") else p.get("x1", p.get("x"))
            self.grouped[name].add(lead.shape[0] if lead.dim() == 4 else lead.numel() // lead.shape[-1])
        ws = None
        if name in ("gemm", "gemm_relu", "wgrad_tn"):  # the split-K workspace: written only by split launches
            ws = self.ops._splitk_buffers(p["a"].device)[0]
            ws.fill_(float("nan"))
        if name == "groupnorm":  # the statistics are checked at every call: ask for them, hand back what was asked
            kwargs = dict(kwargs, want_stats=True)
        ret = real(*args, **kwargs)
        split = ws is not None and bool((ws == ws).any())
        self.split_calls += split
        got = ret
        if name == "groupnorm" and not p["want_stats"]:
            ret = ret[:-1] if p["want_raw"] else ret[0]
        shape, plan = _describe(name, p)
        if ws is not None:
            plan += " split=" + ("k" if split else "1")
        if aliased:
            shape += " alias:" + "+".join(aliased)
        site = _call_site()
        self._abs = 0.0
        try:
            err = self._compare(name, p, sub, got)
        except AssertionError as e:
            self.failures.append((name, site, f"{shape} {plan}", str(e)))
            err = math.inf
        key = (name, shape, plan)
        rec = self.records.setdefault(key, [0, 0.0, site, 0.0])
        rec[0] += 1
        if err > rec[1]:
            rec[1], rec[2] = err, site
        rec[3] = max(rec[3], self._abs)
        return ret

    # -------------------------------------------------------------------------------------------------- comparisons
    def _close(self, name, got, ref, what, bound=None):
        tol, nrel = bound or BOUNDS[name]
        d = (got.detach().float() - ref.detach().float()).abs().max().item()
        self._abs = max(self._abs, d / (ref.detach().float().abs().max().item() + 1e-6))  # the report's "abs" figure
        return close(got, ref, tol=tol, nrel=nrel, what=what)

    @staticmethod
    def _exact(got, ref, what):
        """bit-equal, or an error naming how many elements differ and the first of them"""
        assert got.shape == ref.shape and got.dtype == ref.dtype, \
            f"{what}: {tuple(got.shape)} {got.dtype} vs {tuple(ref.shape)} {ref.dtype}"
        bad = got != ref
        if bad.any():
            i = tuple(bad.nonzero()[0].tolist())
            raise AssertionError(f"{what}: {int(bad.sum())} of {bad.numel()} elements differ, the first at {list(i)}: "
                                 f"{got[i].item():g} vs {ref[i].item():g}")
        return 0.0

    def _compare(self, name, p, sub, got):
        torch.cuda.synchronize()
        ref = getattr(R, name)(**(dict(sub, want_stats=True) if name == "groupnorm" else sub))
        if name in ("gemm", "gemm_relu"):
            return self._compare_gemm(p, got, ref, name)
        if name in EXACT:
            return self._exact(got, ref, "out")
        if name in ("softmax_rows", "weighted_sum", "gaussian_sample"):
            return self._close(name, got, ref, "out")
        if name == "instance_norm":
            return max(self._close(name, got[i], ref[i], f"y image {i}") for i in range(got.shape[0]))
        if name == "lineart_out":
            (y, u8), (ref_y, ref_u8) = (got, ref) if p["want_u8"] else ((got, None), (ref, None))
            err = max(self._close(name, y[i], ref_y[i], f"y image {i}") for i in range(y.shape[0]))
            if u8 is not None:
                self._exact(u8, R._quantise(y[:, 0]), "u8 against the quantised y")
                d = (u8.int() - ref_u8.int()).abs().max().item()
                assert d <= 1, f"u8 {d} levels from the quantised reference"
            return err
        if name == "hed_side_pool":
            err = self._close(name, got[0], ref[0], "side")
            if p["pool"]:
                self._exact(got[1], ref[1], "pooled")
            return err
        if name == "groupnorm":
            outs = list(got)
            errs = [self._close_grouped(name, outs[0], ref[0], p["gamma_hi"] is not None, "y")]
            if p["want_raw"]:
                errs.append(self._close(name, outs[1], ref[1], "raw"))
            b = p["x1"].shape[0]
            st, st_ref = outs[-1].view(b, -1, 2), ref[-1].view(b, -1, 2)
            errs += [self._close(name, st[..., i], st_ref[..., i], f"stats {w}", GN_STATS) for i, w in ((0, "sum"), (1, "sumsq"))]
            return max(errs)
        if name == "layernorm":
            return self._close_grouped(name, got.reshape(-1, got.shape[-1]), ref.reshape(-1, ref.shape[-1]),
                                       p["gamma_hi"] is not None, "y")
        if name == "attention":
            ref_o, ref_lse = (ref, None) if p["lse"] is None else ref
            err = self._close_per_image(name, got, ref_o, p["batch"], "out")
            if ref_lse is not None:
                d = (p["lse"] - ref_lse).abs().max().item()
                assert d <= LSE_ABS * max(1.0, ref_lse.abs().max().item()), f"lse max err {d:.3e}"
            nk, vt = p["nk"], p["vt"]
            assert (vt[..., nk:] == 0).all(), "V^T key padding [nk, tok_pad) is not zero"
            return err
        if name == "wgrad_tn":
            return self._close(name, got, ref, "dW")
        if name == "attention_bwd":
            errs = [self._close_per_image(name, got[2], ref[2], p["batch"], "dv")]
            errs += [self._close_per_image(name, g, r, p["batch"], w, ATTN_DQK) for g, r, w in zip(got, ref, ("dq", "dk"))]
            given_o = R.attention_dqk_given_o(*(p[k] for k in ("q", "k", "v", "o", "dout", "batch", "heads", "nq", "nk",
                                                             "head_dim")))
            for g, r, w in zip(got, given_o, ("dq", "dk")):
                self._close_per_image(name, g, r, p["batch"], f"{w} (row term from o)", ATTN_DQK_GIVEN_O)
            return max(errs)
        if name == "groupnorm_bwd":
            dx1, dx2 = got if p["want_dx2"] else (got, None)
            errs = [self._close(name, dx1, ref[0], "dx1")]
            if dx2 is not None:
                errs.append(self._close(name, dx2, ref[1], "dx2"))
            for t, r, w in ((p["dgamma"], ref[2], "dgamma"), (p["dbeta"], ref[3], "dbeta")):
                if t is not None:
                    errs.append(self._close(name, t, r, w))
            return max(errs)
        if name == "layernorm_bwd":
            errs = [self._close(name, got, ref[0], "dx")]
            for t, r, w in ((p["dgamma"], ref[1], "dgamma"), (p["dbeta"], ref[2], "dbeta")):
                if t is not None:
                    errs.append(self._close(name, t, r, w))
            return max(errs)
        raise AssertionError(f"no comparison for {name}")

    def _close_grouped(self, name, got, ref, grouped, what):
        if not grouped:
            return self._close(name, got, ref, what)
        return max(self._close(name, g, r, f"{what} {half}") for (half, g), (_, r) in zip(_halves(got), _halves(ref)))

    def _close_per_image(self, name, got, ref, batch, what, bound=None):
        """an attention result of [batch * n, heads * d] per image: a wrong image or head shows however many there are"""
        g, r = got.reshape(batch, -1, got.shape[-1]), ref.reshape(batch, -1, ref.shape[-1])
        return max(self._close(name, g[i], r[i], f"{what} image {i}", bound) for i in range(batch))

    def _compare_gemm(self, p, got, ref, name="gemm"):
        grouped = p["hi"] is not None
        if p["seg_outs"] is None:
            return self._close_grouped(name, got, ref, grouped, "out")
        rpi = p["rows_per_img"]
        outs = list(p["seg_outs"]) + ([p["dup_out"]] if p["dup_out"] is not None else [])
        errs = []
        for i, (g, r) in enumerate(zip(outs, ref)):
            transposed = i < len(p["seg_outs"]) and p["transposed"][i]
            if transposed:  # only the tokens below rows_per_img are written
                g = g.reshape(g.shape[0], -1, g.shape[-1])[..., :rpi]
                r = r.reshape(r.shape[0], -1, r.shape[-1])[..., :rpi]
            what = f"segment {i}" if i < len(p["seg_outs"]) else "dup_out"
            errs.append(self._close_grouped(name, g, r, grouped, what))
        return max(errs)

    # ------------------------------------------------------------------------------------------------------ report
    def report(self, scenario):
        print(f"\n== {scenario}: {sum(self.calls.values())} ops calls, {sum(r[0] for r in self.records.values())} checked, "
              f"{len(self.records)} distinct, {self.split_calls} split-K launches")
        for (op, shape, plan), (n, err, site, mabs) in self.records.items():
            print(f"  {op:14s} {shape:70s} {plan:24s} x{n:<4d} err {err:.2e} abs {mabs:.2e}  {site}")
        worst, worst_abs = {}, {}
        for (op, _, _), (_, err, _, mabs) in self.records.items():
            worst[op] = max(worst.get(op, 0.0), err)
            worst_abs[op] = max(worst_abs.get(op, 0.0), mabs)
        print("  worst per op: " + ", ".join(f"{op} {e:.2e} (abs {worst_abs[op]:.2e})"
                                             for op, e in sorted(worst.items())))
        print(f"  worst of the scenario: {max(worst.values(), default=0.0):.2e}")

    def check(self, scenario):
        self.report(scenario)
        assert not self.failures, f"{len(self.failures)} call(s) of {scenario} differ from the reference:\n" + \
            "\n".join(f"  {op} at {site}: {shape}: {msg}" for op, site, shape, msg in self.failures[:20])
        unchecked = {n for n in self.calls if n not in self.only}
        missing = sorted(unchecked - set(UNCHECKED))
        assert not missing, f"{scenario} calls ops functions that are neither checked nor listed in UNCHECKED: {missing}"


# -------------------------------------------------------------------------------------------------------- scenarios
class Models:
    """one SD1.5 model (and trainer) at a time: the previous one is freed before the next is built"""

    def __init__(self):
        self.kind, self.obj = None, None

    CONFIGS = {"finetune": None, "pretrain": "ctrlora_pretrain_sd15_9tasks_rank128.yaml",
               "inference_2loras": "ctrlora_inference_sd15_rank128_2loras.yaml"}

    def get(self, kind):
        if kind != self.kind:
            self.free()
            import bench
            cfg = self.CONFIGS[kind] and os.path.join(ROOT, "configs", self.CONFIGS[kind])
            self.obj, self.kind = bench.build_model(torch.device("cuda"), seed=0, config=cfg), kind
        return self.obj

    def free(self):
        self.kind, self.obj = None, None
        gc.collect()
        torch.cuda.empty_cache()


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _randn(g, *shape):
    return torch.randn(*shape, device="cuda", generator=g)


def _signature(members, name):
    """the signature the shadow binds a call of ops.<name> by: gemm_relu takes gemm's arguments through **kwargs"""
    return inspect.signature(members["gemm" if name == "gemm_relu" else name])


def _corrupt_once(real, when, corrupt, sig=None):
    """`real` with the result of its first call that satisfies when(bound arguments) corrupted in Python"""
    state = {"done": False, "sig": sig or inspect.signature(real)}

    def fn(*args, **kwargs):
        p = state["sig"].bind(*args, **kwargs)
        p.apply_defaults()
        p = dict(p.arguments)
        if state["done"] or not when(p):
            return real(*args, **kwargs)
        state["done"] = True
        return corrupt(p, args, kwargs)
    fn.state = state
    return fn


def _assert_reported(sh, op, text=""):
    assert sh.calls[op] > 1
    hits = [f for f in sh.failures if f[0] == op and text in f[3]]
    assert hits, f"the corrupted {op} call was not reported; failures: {sh.failures}"
    assert len({f[1] for f in hits}) == 1, hits  # one call, named by its call site
    print(f"\nreported: {hits[0][0]} at {hits[0][1]}: {hits[0][2]}: {hits[0][3].splitlines()[0]}")
