"""The kernels every training and evaluation loop runs, at every shape the C ABI accepts: Adam (single-tensor and
multi-tensor entry points), the image metrics (PSNR / SSIM / MSE), the frame ray generator and the pixel ray bank.

Each is checked against a float64 evaluation, in numpy, of the formula the kernel restates, with the fp32 constants the
reference code uses, and against the reference as written (CPU torch, the oracle, the host loaders) as a second check.
Every bar sits next to the largest error measured on an H100; each check prints `measured <err> bar <bar>`.
"""
import ctypes as C
import math

import numpy as np
import pytest
import torch

from helpers import oracle

pytestmark = pytest.mark.gpu

import mipnerf_pl_b200 as mp  # noqa: E402
from mipnerf_pl_b200 import _cabi  # noqa: E402
from mipnerf_pl_b200.ops import _stream  # noqa: E402
from mipnerf_pl_b200.rays import BLENDER_CAMERA_ANGLE_X  # noqa: E402

DEV = "cuda:0"
FLT_MIN = float(np.finfo(np.float32).tiny)


def lib():
    return _cabi.lib()


def check(what, err, bar):
    print(f"{what}: measured {err:.3g} bar {bar:.3g}")
    assert err <= bar, f"{what}: {err:.3g} > {bar:.3g}"


def fl32(x):
    return float(np.float32(x))


def ulp32(x):
    """The fp32 spacing at |x| (x float32)."""
    x = np.abs(np.asarray(x, dtype=np.float32))
    return np.spacing(x).astype(np.float64)


def same_class(a, b):
    """NaN where NaN, the same infinities, finite where finite."""
    return (np.array_equal(np.isnan(a), np.isnan(b)) and np.array_equal(np.isposinf(a), np.isposinf(b))
            and np.array_equal(np.isneginf(a), np.isneginf(b)))


def consistent(got, host, ref, scale):
    """The kernel against the reference as written, in units of `scale`: how much further the kernel is from the host
    result than the host is from float64, max(|got - host| - |host - ref|) / scale.  It is at most the kernel's own
    error against float64, so it is held to the same bar."""
    got, host, ref = (np.asarray(x, dtype=np.float64) for x in (got, host, ref))
    excess = (np.abs(got - host) - np.abs(host - ref)) / scale
    return max(float(excess.max()), 0.0) if excess.size else 0.0


# ================================================================================================ Adam
# Per step, both references start from the kernel's own state before the step, so each step's rounding is measured on
# its own and nothing compounds.  Against float64: m and v against torch's formula, and the update p_new - p_old against
# the formula on the kernel's new m and v, with the half ulp the final `p + update` rounding may add taken out.  Errors
# are relative to max(|ref|, scale): m to the larger of |m_old| and |c1 (g - m_old)|, v to max(v, FLT_MIN).
# Against CPU torch.optim.Adam(foreach=False) in fp32 the same relative errors (torch's CPU kernels fuse some of these
# multiply-adds, the library rounds each operation), the update with both parameter roundings taken out.
ADAM_STATE_BAR = 3.6e-7   # m and v: measured 1.6e-7 (m) and 1.7e-7 (v)
ADAM_UPDATE_BAR = 4.8e-7  # update: measured 2.4e-7
TORCH_STATE_BAR = 2.4e-7  # m and v against torch: measured 1.2e-7
TORCH_UPDATE_BAR = 8e-7   # update against torch: measured 3.9e-7

SIZES = (0, 1, 255, 256, 257, 70001)
NONZERO = SIZES[1:]
MODEL_SIZES = tuple(p.numel() for p in mp.MipNerf().parameters())   # the 24 tensors FusedAdam steps in training
# zero-size tensors first, in the middle, last of one launch / first of the next (32 tensors per launch) and last
ZEROS = {33: (0, 16, 31), 65: (0, 32, 40, 64)}


def group_sizes(count):
    if count == 24:
        return list(MODEL_SIZES)
    sizes = [NONZERO[(i + 2) % len(NONZERO)] for i in range(count)]
    for i in ZEROS.get(count, ()):
        sizes[i] = 0
    return sizes


def adam_state_f64(m, v, g, betas, grad_scale):
    """torch's single-tensor Adam state update (torch/optim/adam.py, foreach=False) in float64: lerp weight
    fl32(1 - b1), mul fl32(b2), addcmul value fl32(1 - b2) -- the scalars torch hands its fp32 kernels, each rounded
    once from double."""
    b1, b2 = betas
    c1, c2 = fl32(1 - b1), fl32(1 - b2)
    g = g.astype(np.float64) * grad_scale
    m, v = m.astype(np.float64), v.astype(np.float64)
    with np.errstate(over="ignore", invalid="ignore"):
        return m + c1 * (g - m), fl32(b2) * v + c2 * g * g


def adam_update_f64(m_new, v_new, lr, betas, eps, step):
    """-step_size m / (sqrt(v) / sqrt(1 - b2^t) + eps) with step_size = lr / (1 - b1^t): the bias corrections in
    double, rounded to fp32 where torch passes them to its kernels."""
    b1, b2 = betas
    step_size = fl32(lr / (1 - b1 ** step))
    bc2_sqrt = fl32(math.sqrt(1 - b2 ** step))
    with np.errstate(over="ignore", invalid="ignore", divide="ignore"):
        return -step_size * m_new.astype(np.float64) / (np.sqrt(v_new.astype(np.float64)) / bc2_sqrt + fl32(eps))


def torch_adam_step(p0, m0, v0, g, lr, betas, eps, step, grad_scale):
    """One CPU torch.optim.Adam(foreach=False) step from the given fp32 state (step = the count after it)."""
    t = torch.nn.Parameter(torch.from_numpy(p0.copy()))
    opt = torch.optim.Adam([t], lr=lr, betas=betas, eps=eps, foreach=False)
    if step > 1:
        opt.state[t] = {"step": torch.tensor(float(step - 1)), "exp_avg": torch.from_numpy(m0.copy()),
                        "exp_avg_sq": torch.from_numpy(v0.copy())}
    t.grad = torch.from_numpy(g.copy()) * grad_scale
    opt.step()
    return t.detach().numpy(), opt.state[t]["exp_avg"].numpy(), opt.state[t]["exp_avg_sq"].numpy()


def adam_errors(p0, m0, v0, g, p1, m1, v1, lr, betas, eps, step, grad_scale, tag):
    """One tensor's step (fp32 numpy before / after) against float64 and CPU torch; asserts that every non-finite value
    matches torch's class and returns the largest errors over the finite ones."""
    tp, tm, tv = torch_adam_step(p0, m0, v0, g, lr, betas, eps, step, grad_scale)
    for name, got, want in (("exp_avg", m1, tm), ("exp_avg_sq", v1, tv), ("param", p1, tp)):
        assert same_class(got, want), f"{tag}: {name} is not in the non-finite class torch gives"
    m_ref, v_ref = adam_state_f64(m0, v0, g, betas, grad_scale)
    d_ref = adam_update_f64(m1, v1, lr, betas, eps, step)
    d_got = p1.astype(np.float64) - p0.astype(np.float64)
    d_torch = tp.astype(np.float64) - p0.astype(np.float64)
    fin = np.isfinite(tm) & np.isfinite(tv) & np.isfinite(tp)   # elsewhere the class check above is the comparison
    c1 = fl32(1 - betas[0])
    with np.errstate(over="ignore", invalid="ignore"):
        m_scale = np.maximum(np.abs(m0.astype(np.float64)), np.abs(c1 * (g.astype(np.float64) * grad_scale - m0)))
        em = np.abs(m1 - m_ref) / np.maximum(np.maximum(np.abs(m_ref), m_scale), FLT_MIN)
        ev = np.abs(v1 - v_ref) / np.maximum(v_ref, FLT_MIN)
        ed = np.maximum(np.abs(d_got - d_ref) - 0.5 * ulp32(p1), 0) / np.maximum(np.abs(d_ref), FLT_MIN)
        # torch's update starts from its own m, which may sit an ulp of m_scale away: the update's scale is m_scale's
        d_scale = np.maximum(np.abs(d_ref), np.abs(adam_update_f64(m_scale, v1, lr, betas, eps, step)))
        et = np.maximum(np.abs(d_got - d_torch) - ulp32(p1), 0) / np.maximum(d_scale, FLT_MIN)
        m_den = np.maximum(np.maximum(np.abs(tm), m_scale), FLT_MIN)
        etm = np.maximum(np.abs(m1 - tm) / m_den, np.abs(v1 - tv) / np.maximum(tv, FLT_MIN))
    if not fin.any():
        return dict(m=0.0, v=0.0, d=0.0, torch_mv=0.0, torch_d=0.0)
    return dict(m=float(em[fin].max()), v=float(ev[fin].max()), d=float(ed[fin].max()),
                torch_mv=float(etm[fin].max()), torch_d=float(et[fin].max()))


def merge(worst, errs):
    for k, e in errs.items():
        worst[k] = max(worst.get(k, 0), e)


def report(worst, tag):
    check(f"{tag}: exp_avg_sq vs float64 (rel)", worst["v"], ADAM_STATE_BAR)
    check(f"{tag}: exp_avg vs float64 (rel)", worst["m"], ADAM_STATE_BAR)
    check(f"{tag}: update vs float64 (rel)", worst["d"], ADAM_UPDATE_BAR)
    check(f"{tag}: exp_avg / exp_avg_sq vs torch (rel)", worst["torch_mv"], TORCH_STATE_BAR)
    check(f"{tag}: update vs torch (rel)", worst["torch_d"], TORCH_UPDATE_BAR)


def random_grads(sizes, gen):
    """Normal gradients at a random scale 1e-6 .. 10 per tensor and step."""
    return [torch.randn(n, generator=gen).numpy() * 10.0 ** int(torch.randint(-6, 2, (1,), generator=gen))
            for n in sizes]


class AdamGroup:
    """fp32 device tensors of one optimiser group, stepped through either C-ABI entry point."""

    def __init__(self, sizes, seed, resume=False):
        gen = torch.Generator().manual_seed(seed)
        self.sizes = list(sizes)
        self.p = [(1e-3 * torch.randn(n, generator=gen)).to(DEV) for n in sizes]
        self.m = [(1e-2 * torch.randn(n, generator=gen) if resume else torch.zeros(n)).to(DEV) for n in sizes]
        self.v = [(1e-4 * torch.rand(n, generator=gen) if resume else torch.zeros(n)).to(DEV) for n in sizes]
        self.g = [torch.zeros(n, device=DEV) for n in sizes]

    def state(self):
        return [[t.cpu().numpy().copy() for t in ts] for ts in (self.p, self.m, self.v)]

    def step(self, entry, grads, lr, betas, eps, step, grad_scale):
        for dst, src in zip(self.g, grads):
            dst.copy_(torch.from_numpy(src))
        n, st = len(self.sizes), _stream(torch.device(DEV))
        if entry == "multi":
            ptrs = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts]) if n else None  # noqa: E731
            rc = lib().mipnerf_b200_adam_step_multi(n, ptrs(self.p), ptrs(self.g), ptrs(self.m), ptrs(self.v),
                                                    (C.c_int64 * n)(*self.sizes) if n else None, lr, betas[0],
                                                    betas[1], eps, step, grad_scale, st)
            assert rc == _cabi.OK, _cabi.last_error()
        else:
            for p, g, m, v, size in zip(self.p, self.g, self.m, self.v, self.sizes):
                rc = lib().mipnerf_b200_adam_step(p.data_ptr(), g.data_ptr(), m.data_ptr(), v.data_ptr(), size, lr,
                                                  betas[0], betas[1], eps, step, grad_scale, st)
                assert rc == _cabi.OK, _cabi.last_error()
        torch.cuda.synchronize()


def run_adam(group, entry, steps, lr=1e-3, betas=(0.9, 0.999), eps=1e-8, grad_scale=1.0, first_step=1, seed=0,
             grads=None, check_every=1):
    """`steps` steps from step count `first_step`, every `check_every`-th (and the first and last) checked."""
    gen = torch.Generator().manual_seed(1000 + seed)
    worst = {}
    for k in range(steps):
        step = first_step + k
        gs = grads(k) if grads else random_grads(group.sizes, gen)
        checked = k == 0 or k == steps - 1 or k % check_every == 0
        if checked:
            p0, m0, v0 = group.state()
        group.step(entry, gs, lr, betas, eps, step, grad_scale)
        if checked:
            p1, m1, v1 = group.state()
            for i, g in enumerate(gs):
                merge(worst, adam_errors(p0[i], m0[i], v0[i], g, p1[i], m1[i], v1[i], lr, betas, eps, step, grad_scale,
                                         f"tensor {i} (n={group.sizes[i]}) step {step}"))
    return worst


@pytest.mark.parametrize("grad_scale", [1.0, 0.25])
@pytest.mark.parametrize("entry", ["multi", "single"])
@pytest.mark.parametrize("count", [0, 1, 24, 33, 65])
def test_adam_tensor_counts_and_sizes(count, entry, grad_scale):
    """0 / 1 / the model's 24 / 33 and 65 tensors (two and three launches of the multi-tensor entry), sizes 0, 1, 255,
    256, 257 and 70001 with zero-size tensors first, in the middle and last: two steps from zero state."""
    group = AdamGroup(group_sizes(count), seed=count)
    worst = run_adam(group, entry, 2, grad_scale=grad_scale, seed=count)
    if count:
        report(worst, f"count={count} {entry} grad_scale={grad_scale}")


@pytest.mark.parametrize("entry", ["multi", "single"])
def test_adam_long_run(entry):
    """1000 steps: bias corrections up to 1 - 0.999^1000 (every 50th step and the last checked)."""
    worst = run_adam(AdamGroup(SIZES, seed=7), entry, 1000, seed=7, check_every=50)
    report(worst, f"1000 steps {entry}")


@pytest.mark.parametrize("entry", ["multi", "single"])
def test_adam_resumed_state_and_other_hyperparameters(entry):
    """A state resumed at step 37 (what loading a checkpoint gives), then betas (0.5, 0.99) with eps 1e-15 -- where
    the lerp weight 1 - b1 is 0.5 and eps sits below the smallest denominators."""
    worst = run_adam(AdamGroup(SIZES, seed=3, resume=True), entry, 3, first_step=38, seed=3, lr=5e-4)
    report(worst, f"resumed at step 37 {entry}")
    worst = run_adam(AdamGroup(SIZES, seed=4), entry, 3, betas=(0.5, 0.99), eps=1e-15, seed=4)
    report(worst, f"betas (0.5, 0.99) eps 1e-15 {entry}")
    worst = run_adam(AdamGroup(SIZES, seed=5, resume=True), entry, 2, betas=(0.5, 0.99), eps=1e-15, first_step=38,
                     grad_scale=0.25, seed=5)
    report(worst, f"resumed, betas (0.5, 0.99) eps 1e-15 grad_scale 0.25 {entry}")


SPECIAL = {  # gradient value -> what it exercises
    0.0: "zero: update -lr m / eps while v is 0",
    1e-25: "tiny: (1 - b2) g g underflows to 0",
    3e19: "huge: g g overflows fp32, (1 - b2) g g does not",
    -3e19: "huge, negative",
    1e21: "huger: (1 - b2) g g overflows too",
    float("nan"): "NaN",
    float("inf"): "inf",
}


@pytest.mark.parametrize("entry", ["multi", "single"])
def test_adam_special_gradients(entry):
    """Zero, tiny, huge, infinite and NaN gradients, from zero state and from a resumed state with exp_avg set and
    exp_avg_sq zero: every result in torch's non-finite class, the finite ones on the float64 bars."""
    vals = np.array(list(SPECIAL), dtype=np.float32)
    n = 256 * len(vals)
    for resume in (False, True):
        group = AdamGroup([n, 1], seed=11, resume=resume)
        if resume:
            group.v[0].zero_()
        grads = lambda k: [np.repeat(vals, 256) * np.float32(1 + k), np.zeros(1, np.float32)]  # noqa: E731
        worst = run_adam(group, entry, 2, first_step=38 if resume else 1, grads=grads)
        report(worst, f"special gradients {entry} {'resumed' if resume else 'from zero'}")
        p = group.p[0].cpu().numpy().reshape(len(vals), 256)
        assert np.isnan(p[np.isnan(vals)]).all() and np.isnan(p[np.isinf(vals)]).all()


def test_fused_adam_grouped_and_per_tensor_paths_agree():
    """FusedAdam's one-launch group path and its per-tensor fallback give bit-identical parameters and state."""
    def run(fallback, grad_scale):
        gen = torch.Generator().manual_seed(21)
        ps = [torch.nn.Parameter((1e-2 * torch.randn(n, generator=gen)).to(DEV)) for n in group_sizes(33) if n]
        opt = mp.FusedAdam(ps, lr=1e-3, grad_scale=grad_scale)
        if fallback:
            opt._step_group = lambda *a: False
        for _ in range(3):
            for p in ps:
                p.grad = torch.randn(p.shape, generator=gen).to(DEV)
            opt.step()
        torch.cuda.synchronize()
        return [t.cpu() for p in ps for t in (p.detach(), opt.state[p]["exp_avg"], opt.state[p]["exp_avg_sq"])]
    for grad_scale in (1.0, 0.25):
        for a, b in zip(run(False, grad_scale), run(True, grad_scale)):
            assert torch.equal(a, b)


def test_adam_multi_refusal_leaves_every_tensor_untouched():
    """A negative size in the second launch's tensors is refused before the first launch runs."""
    group = AdamGroup(group_sizes(33), seed=2)
    for g in group.g:
        g.fill_(1.0)
    before = group.state()
    n = 33
    sizes = list(group.sizes)
    sizes[32] = -1
    ptrs = lambda ts: (C.c_void_p * n)(*[t.data_ptr() for t in ts])  # noqa: E731
    rc = lib().mipnerf_b200_adam_step_multi(n, ptrs(group.p), ptrs(group.g), ptrs(group.m), ptrs(group.v),
                                            (C.c_int64 * n)(*sizes), 1e-3, 0.9, 0.999, 1e-8, 1, 1.0,
                                            _stream(torch.device(DEV)))
    assert rc == _cabi.EINVAL and b"tensor 32" in lib().mipnerf_b200_last_error()
    torch.cuda.synchronize()
    for a, b in zip(before, group.state()):
        for x, y in zip(a, b):
            assert np.array_equal(x, y)


# ================================================================================================ image metrics
# float64 PSNR / SSIM / MSE with the reference's fp32 Gaussian window (oracle.gaussian_window), zero padding,
# C1 = 0.01^2 and C2 = 0.03^2 (utils/metrics.py:44-126, 182-197).  Both fp32 implementations (the kernel and the
# oracle, which is the reference as written) compute sigma^2 as E[x^2] - mu^2 and lose digits where sigma^2 << mu^2:
# constant images and flat bright ones (0.98 +- 1e-3) have their own SSIM bar.
PSNR_BAR = 2.4e-7       # relative: measured 1.1e-7
MSE_BAR = 1.6e-7        # relative: measured 8.2e-8
SSIM_BAR = 1.2e-7       # absolute, on the mean: measured 6.0e-8
FLAT_SSIM_BAR = 1.2e-5  # absolute, constant and flat bright images: measured 5.3e-6 (the oracle: 1.1e-4)

METRIC_SHAPES = [(1, 1, 3), (1, 37, 3), (5, 5, 3), (10, 11, 1), (15, 17, 4), (16, 16, 3), (17, 33, 3), (3, 2000, 3),
                 (2000, 3, 3), (1100, 1100, 3)]
CONTENTS = ["random", "noisy", "identical", "constant", "flat_bright", "out_of_range"]


def metric_images(shape, content, seed):
    rng = np.random.default_rng(seed)
    a = rng.random(shape, dtype=np.float32)
    if content == "random":
        b = rng.random(shape, dtype=np.float32)
    elif content == "noisy":
        b = np.clip(a + 0.05 * rng.standard_normal(shape), 0, 1).astype(np.float32)
    elif content == "identical":
        b = a.copy()
    elif content == "constant":
        a, b = np.full(shape, 0.3, np.float32), np.full(shape, 0.7, np.float32)
    elif content == "flat_bright":
        a = (0.98 + 1e-3 * rng.uniform(-1, 1, shape)).astype(np.float32)
        b = (0.98 + 1e-3 * rng.uniform(-1, 1, shape)).astype(np.float32)
    else:
        a = rng.uniform(-0.5, 1.5, shape).astype(np.float32)
        b = (a + 0.3 * rng.standard_normal(shape)).astype(np.float32)
    return a, b


def gauss_filter_f64(x, g):
    """Zero-padded separable 11-tap correlation of [H, W, C] over H and W (F.conv2d(padding=5) with outer(g, g))."""
    h, w = x.shape[:2]
    xp = np.pad(x, ((5, 5), (5, 5), (0, 0)))
    t = sum(g[k] * xp[k:k + h] for k in range(11))
    return sum(g[k] * t[:, k:k + w] for k in range(11))


def metrics_f64(pred, target):
    g = oracle.gaussian_window().numpy().astype(np.float64)
    a, b = pred.astype(np.float64), target.astype(np.float64)
    mu1, mu2 = gauss_filter_f64(a, g), gauss_filter_f64(b, g)
    s11 = gauss_filter_f64(a * a, g) - mu1 * mu1
    s22 = gauss_filter_f64(b * b, g) - mu2 * mu2
    s12 = gauss_filter_f64(a * b, g) - mu1 * mu2
    c1, c2 = 0.01 ** 2, 0.03 ** 2
    ssim = ((2 * mu1 * mu2 + c1) * (2 * s12 + c2)) / ((mu1 * mu1 + mu2 * mu2 + c1) * (s11 + s22 + c2))
    mse = float(np.mean((a - b) ** 2))
    with np.errstate(divide="ignore"):
        psnr = float(-10 * np.log10(mse))
    return psnr, float(ssim.mean()), mse


def device_metrics(pred, target):
    h, w, c = pred.shape
    p, t = torch.from_numpy(pred).to(DEV), torch.from_numpy(target).to(DEV)
    nbytes = lib().mipnerf_b200_image_metrics_scratch_bytes(h, w, c)
    assert nbytes == 16 * ((w + 15) // 16) * ((h + 15) // 16) * c
    scratch = torch.empty(nbytes, dtype=torch.uint8, device=DEV)
    out = torch.empty(3, device=DEV)
    rc = lib().mipnerf_b200_image_metrics(p.data_ptr(), t.data_ptr(), h, w, c, scratch.data_ptr(), nbytes,
                                          out.data_ptr(), _stream(torch.device(DEV)))
    assert rc == _cabi.OK, _cabi.last_error()
    return out.cpu().numpy()


@pytest.mark.parametrize("shape", METRIC_SHAPES, ids=lambda s: "x".join(map(str, s)))
def test_image_metrics_against_float64(shape):
    """Images smaller than a 16x16 tile or the 11-pixel window, 1 and 4 channels, thin frames, and 1100x1100 (5041
    partial blocks per channel, past the reduce kernel's 1024 threads), with every content."""
    for content in CONTENTS:
        pred, target = metric_images(shape, content, seed=sum(shape))
        tag = f"{'x'.join(map(str, shape))} {content}"
        got = device_metrics(pred, target)
        again = device_metrics(pred, target)
        assert np.array_equal(got.view(np.int32), again.view(np.int32)), f"{tag}: not bit-reproducible"
        psnr, ssim, mse = metrics_f64(pred, target)
        o_psnr, o_ssim = (float(x) for x in oracle.eval_errors(torch.from_numpy(pred)[None],
                                                                torch.from_numpy(target)[None]))
        if content == "identical":
            # the reference gives exactly these: mse 0, ssim_map x / x = 1 everywhere
            assert got[0] == np.inf and got[1] == 1.0 and got[2] == 0.0, (tag, got)
            assert o_psnr == np.inf and o_ssim == 1.0
            continue
        check(f"{tag}: psnr vs float64 (rel)", abs(got[0] - psnr) / abs(psnr), PSNR_BAR)
        check(f"{tag}: mse vs float64 (rel)", abs(got[2] - mse) / mse, MSE_BAR)
        bar = FLAT_SSIM_BAR if content in ("constant", "flat_bright") else SSIM_BAR
        check(f"{tag}: ssim vs float64 (abs)", abs(got[1] - ssim), bar)
        if bar == FLAT_SSIM_BAR:
            print(f"{tag}: ssim vs float64, oracle (fp32 torch) {abs(o_ssim - ssim):.3g}, kernel {abs(got[1] - ssim):.3g}")
        check(f"{tag}: psnr vs oracle", consistent(got[0], o_psnr, psnr, abs(psnr)), PSNR_BAR)
        check(f"{tag}: ssim vs oracle", consistent(got[1], o_ssim, ssim, 1.0), bar)


def test_ssim_wrapper_equals_eval_errors():
    pred, target = metric_images((37, 29, 3), "noisy", seed=1)
    p, t = torch.from_numpy(pred)[None].to(DEV), torch.from_numpy(target)[None].to(DEV)
    psnr, ssim = mp.eval_errors(p, t)
    assert float(mp.ssim(p.permute(0, 3, 1, 2), t.permute(0, 3, 1, 2))) == float(ssim)
    assert np.array_equal(device_metrics(pred, target)[:2], np.array([float(psnr), float(ssim)], np.float32))


# ================================================================================================ ray generator
# float64 of ray_kernels.cu's pinhole formulas on the fp32 pose and focal:
#   d = R ((x - W/2 + .5) / f, -(y - H/2 + .5) / f, -1),  viewdir = d / |d|,  radius = |R[:, 1]| / f * 2 / sqrt(12).
# Direction errors are per ray, relative to |d|.
DIR_BAR = 3.2e-7      # directions: measured 1.6e-7 (both kernels)
VIEWDIR_BAR = 3.6e-7  # viewdirs, absolute: measured 1.7e-7
RADIUS_BAR = 3e-7     # radii, relative: measured 1.4e-7
NARROW, WIDE = 1e-3, 3.0   # camera_angle_x: focal 500 W (large) and 0.035 W (small)


def rotation(seed):
    q, r = np.linalg.qr(np.random.default_rng(seed).standard_normal((3, 3)))
    return q * np.sign(np.diag(r))


POSES = {"spheric": mp.spheric_pose(0.7),
         "far": np.concatenate([rotation(5), [[3.0e4], [-1.7e4], [9.0e3]]], 1).astype(np.float32)}


def rays_f64(c2w, h, w, focal, row0, rows):
    c2w = np.asarray(c2w, dtype=np.float32).astype(np.float64)
    focal = float(np.float32(focal))
    y, x = np.meshgrid(np.arange(row0, row0 + rows, dtype=np.float64), np.arange(w, dtype=np.float64), indexing="ij")
    cam = np.stack([(x - w * 0.5 + 0.5) / focal, -(y - h * 0.5 + 0.5) / focal, -np.ones_like(x)], -1)
    d = (cam @ c2w[:, :3].T).reshape(-1, 3)
    radius = np.linalg.norm(c2w[:, 1]) / focal * 2 / np.sqrt(12)
    return d, d / np.linalg.norm(d, axis=-1, keepdims=True), radius


def np_rays(rays):
    return mp.Rays(*[f.cpu().numpy() for f in rays])


def check_frame(tag, got, c2w, h, w, focal, row0=0, rows=None):
    rows = h - row0 if rows is None else rows
    d, vd, radius = rays_f64(c2w, h, w, focal, row0, rows)
    dn = np.linalg.norm(d, axis=-1)
    check(f"{tag}: directions vs float64", float((np.abs(got.directions - d).max(-1) / dn).max()), DIR_BAR)
    check(f"{tag}: viewdirs vs float64", float(np.abs(got.viewdirs - vd).max()), VIEWDIR_BAR)
    check(f"{tag}: radii vs float64", float(np.abs(got.radii / radius - 1).max()), RADIUS_BAR)
    assert np.array_equal(got.origins, np.broadcast_to(np.asarray(c2w, np.float32)[:, 3], got.origins.shape))
    return d, vd, radius


@pytest.mark.parametrize("pose", list(POSES))
@pytest.mark.parametrize("angle", [BLENDER_CAMERA_ANGLE_X, NARROW, WIDE], ids=["blender", "narrow", "wide"])
@pytest.mark.parametrize("hw", [(2, 1), (3, 5), (7, 800), (801, 799)], ids=lambda s: "x".join(map(str, s)))
def test_generate_rays_frames(hw, angle, pose):
    h, w = hw
    c2w = POSES[pose]
    focal = float(np.float32(0.5 * w / np.tan(0.5 * angle)))
    got = np_rays(mp.generate_rays(c2w, h, w, camera_angle_x=angle, near=2.0, far=6.0, device=DEV))
    tag = f"{h}x{w} {pose} f={focal:.3g}"
    d, vd, radius = check_frame(tag, got, c2w, h, w, focal)
    assert (got.near == 2.0).all() and (got.far == 6.0).all() and (got.lossmult == 1.0).all()
    rad = got.radii.reshape(h, w)
    assert np.array_equal(rad[-1], rad[-2])   # the last row repeats the previous one
    if h < 3:
        return   # the reference's last-row rule (dx[-2:-1]) has no row to repeat at H = 2
    host = mp.blender_rays(c2w, h, w, near=2.0, far=6.0, camera_angle_x=angle)
    hd, hv, hr = (host.directions.reshape(-1, 3), host.viewdirs.reshape(-1, 3), host.radii.reshape(-1))
    dn = np.linalg.norm(d, axis=-1, keepdims=True)
    check(f"{tag}: directions vs blender_rays", consistent(got.directions, hd, d, dn), DIR_BAR)
    check(f"{tag}: viewdirs vs blender_rays", consistent(got.viewdirs, hv, vd, 1.0), VIEWDIR_BAR)
    # the host's finite difference of fp32 directions carries cancellation noise; the kernel's radius is analytic
    check(f"{tag}: radii vs blender_rays", consistent(got.radii.reshape(-1), hr, radius, radius), RADIUS_BAR)
    assert np.array_equal(got.origins, host.origins.reshape(-1, 3))


@pytest.mark.parametrize("shards", [1, 2, 5, 37, 40])
def test_generate_rays_row_shards_equal_the_full_frame(shards):
    """Each rank's rows (render.shard_rows, what multi-GPU rendering asks for), concatenated, are the full frame bit
    for bit; ranks beyond the row count get rows = 0, which is accepted."""
    h, w = 37, 53
    for pose, c2w in POSES.items():
        full = mp.generate_rays(c2w, h, w, device=DEV)
        parts = [mp.generate_rays(c2w, h, w, rows=mp.shard_rows(h, shards, r), device=DEV) for r in range(shards)]
        for k, f in enumerate(full):
            cat = torch.cat([p[k] for p in parts]).cpu().numpy()
            assert np.array_equal(cat.view(np.int32), f.cpu().numpy().view(np.int32)), (pose, shards, k)
        check_frame(f"37x53 {pose} {shards} shards", np_rays(full), c2w, h, w,
                    0.5 * w / np.tan(0.5 * BLENDER_CAMERA_ANGLE_X))
    empty = mp.generate_rays(POSES["far"], h, w, rows=(h, h), device=DEV)
    assert all(f.shape[0] == 0 for f in empty)


# ================================================================================================ pixel ray bank
# float64 of rays_from_pixels_kernel's formulas on the fp32 camera table: image = upper_bound(offsets, id) - 1,
# cam = pix2cam (x + .5, y + .5, 1), d = R cam, radius = |R pix2cam[:, 1]| * 2 / sqrt(12).  The generator's bars.


@pytest.fixture(scope="module")
def bank_scene():
    """About 300 images of random sizes 1..40 (1x1, 1-wide and 1-high ones included), each with its own focal and
    pose, in load_blender_scene's layout (pix2cam maps (x + .5, y + .5, 1) to the camera direction)."""
    rng = np.random.default_rng(17)
    n = 301
    hs, ws = rng.integers(1, 41, n), rng.integers(1, 41, n)
    hs[[0, 150, 300]] = 1
    ws[[0, 150, 300]] = 1
    hs[[10, 11]], ws[[12, 13]] = 1, 1
    images, pix2cam, c2w = [], [], []
    for i in range(n):
        h, w, f = int(hs[i]), int(ws[i]), float(rng.uniform(5, 200))
        images.append(rng.random((h, w, 3), dtype=np.float32))
        pix2cam.append([[1 / f, 0, -0.5 * w / f], [0, -1 / f, 0.5 * h / f], [0, 0, -1]])
        c2w.append(np.concatenate([rotation(100 + i), rng.uniform(-50, 50, (3, 1))], 1))
    scene = mp.Scene(images, np.array(pix2cam), np.array(c2w), rng.uniform(0.5, 4, n), rng.uniform(0, 2, n),
                     rng.uniform(4, 8, n))
    return scene, mp.DeviceRayBank(scene, DEV)


def bank_f64(scene, bank, ids):
    offsets = bank.offsets.cpu().numpy()
    total = int(offsets[-1])
    ids = np.clip(ids, 0, total - 1)
    img = np.searchsorted(offsets, ids, side="right") - 1
    local = ids - offsets[img]
    w = scene.widths[img].astype(np.int64)
    px, py = (local % w) + 0.5, (local // w) + 0.5
    k = scene.pix2cam[img].astype(np.float64)
    m = scene.cam2world[img].astype(np.float64)
    cam = np.einsum("nij,nj->ni", k, np.stack([px, py, np.ones_like(px)], -1))
    d = np.einsum("nij,nj->ni", m[:, :, :3], cam)
    radius = np.linalg.norm(np.einsum("nij,nj->ni", m[:, :, :3], k[:, :, 1]), axis=-1) * 2 / np.sqrt(12)
    return img, ids, d, radius


def bank_rays(bank, ids, rgb=True):
    """mipnerf_b200_rays_from_pixels straight through the C ABI (rgb=False passes NULL for rgb and the atlas)."""
    ids_d = torch.as_tensor(ids, dtype=torch.int64).to(DEV)
    b = ids_d.numel()
    outs = [torch.full((b, c), float("nan"), device=DEV) for c in (3, 3, 3, 1, 1, 1, 1, 3)]
    ptr = lambda t: t.data_ptr() if b else None  # noqa: E731
    rc = lib().mipnerf_b200_rays_from_pixels(
        bank.cam_table.data_ptr(), bank.offsets.data_ptr(), bank.widths.data_ptr(), bank.num_images, ptr(ids_d), b,
        bank.atlas.data_ptr() if rgb else None, *[ptr(t) for t in outs[:7]], ptr(outs[7]) if rgb else None,
        _stream(torch.device(DEV)))
    assert rc == _cabi.OK, _cabi.last_error()
    torch.cuda.synchronize()
    return [t.cpu().numpy() for t in outs]


def bank_ids(offsets, rng):
    total = int(offsets[-1])
    edges = np.concatenate([offsets - 1, offsets])
    out_of_range = np.array([-1, -2, -(1 << 31), -(1 << 40), np.iinfo(np.int64).min, total, total + 1, (1 << 31) - 1,
                             1 << 31, (1 << 31) + 5, 1 << 40, np.iinfo(np.int64).max], dtype=np.int64)
    shuffled = rng.permutation(total)[:3000]
    repeated = np.repeat(rng.integers(0, total, 50), 7)
    return {"edges": edges, "out_of_range": out_of_range, "random": np.concatenate([shuffled, repeated]),
            "one": np.array([int(rng.integers(0, total))]), "none": np.zeros(0, np.int64),
            "count_4097": rng.integers(-100, total + 100, 4097)}


def test_rays_from_pixels_against_float64_and_the_host_loader(bank_scene):
    scene, bank = bank_scene
    offsets = bank.offsets.cpu().numpy()
    total = int(offsets[-1])
    assert total == int((scene.heights.astype(np.int64) * scene.widths).sum())
    per_image = [mp.image_rays(scene, i) for i in range(len(scene))]
    atlas = np.concatenate([im.reshape(-1, 3) for im in scene.images])
    host = {k: np.concatenate([getattr(r, k).reshape(-1, getattr(r, k).shape[-1]) for r in per_image
                               if k != "radii" or r.radii.shape[0] == r.origins.shape[0]])
            for k in mp.Rays_keys}
    # image_rays' finite-difference radius has no neighbour row in a 1-high image: compare radii on the others
    tall = np.repeat(scene.heights > 1, scene.heights.astype(np.int64) * scene.widths)
    host_radius_row = np.cumsum(tall) - 1
    for name, ids in bank_ids(offsets, np.random.default_rng(3)).items():
        o, d, v, rad, lm, nr, fr, rgb = bank_rays(bank, ids)
        o2, d2, v2, rad2, lm2, nr2, fr2, rgb2 = bank_rays(bank, ids, rgb=False)
        for a, b in ((o, o2), (d, d2), (v, v2), (rad, rad2), (lm, lm2), (nr, nr2), (fr, fr2)):
            assert np.array_equal(a, b, equal_nan=True), f"{name}: rgb = NULL changed a ray field"
        assert np.isnan(rgb2).all()
        if not len(ids):
            continue
        img, cl, d_ref, r_ref = bank_f64(scene, bank, ids)
        dn = np.linalg.norm(d_ref, axis=-1)
        check(f"{name}: directions vs float64", float((np.abs(d - d_ref).max(-1) / dn).max()), DIR_BAR)
        check(f"{name}: viewdirs vs float64", float(np.abs(v - d_ref / dn[:, None]).max()), VIEWDIR_BAR)
        check(f"{name}: radii vs float64", float(np.abs(rad[:, 0] / r_ref - 1).max()), RADIUS_BAR)
        assert np.array_equal(o, scene.cam2world[img][:, :, 3])
        assert np.array_equal(lm[:, 0], scene.lossmult[img]) and np.array_equal(nr[:, 0], scene.near[img])
        assert np.array_equal(fr[:, 0], scene.far[img]) and np.array_equal(rgb, atlas[cl])
        # the host loader (datasets.image_rays), as the reference's Dataset would hand these pixels out
        assert np.array_equal(o, host["origins"][cl]) and np.array_equal(lm, host["lossmult"][cl])
        check(f"{name}: directions vs image_rays", consistent(d, host["directions"][cl], d_ref, dn[:, None]),
              DIR_BAR)
        check(f"{name}: viewdirs vs image_rays", consistent(v, host["viewdirs"][cl], d_ref / dn[:, None], 1.0),
              VIEWDIR_BAR)
        t = tall[cl]
        check(f"{name}: radii vs image_rays", consistent(rad[t, 0], host["radii"][host_radius_row[cl[t]], 0], r_ref[t],
                                                         r_ref[t]), RADIUS_BAR)
    # the DeviceRayBank wrapper gives the same rays
    ids = bank_ids(offsets, np.random.default_rng(4))["count_4097"]
    rays, rgb = bank.rays(torch.from_numpy(ids))
    want = bank_rays(bank, ids)
    for a, b in zip(list(rays) + [rgb], want):
        assert np.array_equal(a.cpu().numpy(), b)
