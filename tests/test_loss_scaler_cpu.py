"""Dynamic loss scaling and gradient clipping (CPU tier): a plain-Python restatement of the policy `mm_loss_scale_update`
implements, pinned to sequences derived by hand from DeepSpeed's DynamicLossScaler.update_scale
(consecutive_hysteresis=False) and FP16_Optimizer.unscale_and_clip_grads.  The GPU tests (tests/test_train_fp16_gpu.py)
compare the device kernel against `ScaleRef`, field by field and bit for bit."""
import math

import numpy as np

F32 = np.float32


class ScaleRef:
    """Host restatement of `mm_loss_scale_state` + `mm_loss_scale_update` in fp32 arithmetic (numpy float32 operations
    are IEEE round-to-nearest, as the kernel's intrinsics are)."""

    def __init__(self, initial_scale_power=16, window=1000, hysteresis=2, min_scale=1.0, dynamic=True, max_norm=None):
        self.scale = F32(2.0 ** initial_scale_power) if dynamic else F32(1.0)
        self.window, self.hysteresis, self.min_scale = int(window), int(hysteresis), F32(min_scale)
        self.dynamic, self.max_norm = dynamic, max_norm
        self.cur_iter, self.last_overflow_iter, self.cur_hysteresis = 0, -1, int(hysteresis)
        self.skip, self.skipped, self.step = 0, 0, 0
        self.grad_mult = F32(1.0) / self.scale

    def update(self, sumsq) -> None:
        ss = F32(sumsq)
        S = self.scale
        overflow = not np.isfinite(ss)
        mult = F32(1.0) / S
        if not overflow and self.max_norm:
            norm = F32(np.sqrt(ss)) / S
            c = (norm + F32(1e-6)) / F32(self.max_norm)
            mult = F32(1.0) / (S * max(c, F32(1.0)))
        self.grad_mult = F32(mult)
        self.skip = int(overflow)
        if overflow:
            self.skipped += 1
        else:
            self.step += 1
        if self.dynamic:
            if overflow:
                if self.hysteresis == 1 or self.cur_hysteresis == 1:
                    self.scale = max(F32(S * F32(0.5)), self.min_scale)
                else:
                    self.cur_hysteresis -= 1
                self.last_overflow_iter = self.cur_iter
            elif (self.cur_iter - self.last_overflow_iter) % self.window == 0:
                self.cur_hysteresis = self.hysteresis
                self.scale = F32(S * F32(2.0))
        self.cur_iter += 1

    def fields(self) -> dict:
        return dict(scale=float(self.scale), cur_iter=self.cur_iter, last_overflow_iter=self.last_overflow_iter,
                    cur_hysteresis=self.cur_hysteresis, skip=self.skip, grad_mult=float(self.grad_mult),
                    skipped=self.skipped, step=self.step)


INF = float("inf")


def _run(ref, pattern):
    scales = []
    for ovf in pattern:
        ref.update(INF if ovf else 1.0)
        scales.append(float(ref.scale))
    return scales


def test_first_overflow_only_consumes_hysteresis():
    r = ScaleRef(initial_scale_power=4, window=4, hysteresis=2)
    r.update(INF)
    assert (float(r.scale), r.cur_hysteresis, r.last_overflow_iter, r.cur_iter) == (16.0, 1, 0, 1)
    assert r.skip == 1 and r.skipped == 1 and r.step == 0


def test_second_consecutive_overflow_halves():
    r = ScaleRef(initial_scale_power=4, window=4, hysteresis=2)
    assert _run(r, [1, 1]) == [16.0, 8.0]
    assert r.last_overflow_iter == 1 and r.skipped == 2


def test_overflow_after_clean_step_halves_again():
    """consecutive_hysteresis=False: a clean step does not restore the hysteresis, so the next overflow halves at once."""
    r = ScaleRef(initial_scale_power=4, window=4, hysteresis=2)
    assert _run(r, [1, 1, 0, 1]) == [16.0, 8.0, 8.0, 4.0]
    assert r.cur_hysteresis == 1 and r.step == 1 and r.skipped == 3


def test_growth_after_window_small():
    """Window 4: after the overflow at iteration 3 the scale doubles at iteration 7 ((7 - 3) % 4 == 0), which also
    restores the hysteresis; the next overflow is absorbed by it."""
    r = ScaleRef(initial_scale_power=4, window=4, hysteresis=2)
    s = _run(r, [1, 1, 0, 1, 0, 0, 0, 0, 1])
    assert s == [16.0, 8.0, 8.0, 4.0, 4.0, 4.0, 4.0, 8.0, 8.0]
    assert r.cur_hysteresis == 1 and r.last_overflow_iter == 8


def test_growth_default_window():
    """Default window 1000 and no overflow: the first doubling is at iteration 999 ((999 - (-1)) % 1000 == 0), the next
    at 1999."""
    r = ScaleRef()
    s = _run(r, [0] * 2000)
    assert s[998] == 65536.0 and s[999] == 131072.0 and s[1998] == 131072.0 and s[1999] == 262144.0
    assert r.step == 2000 and r.skipped == 0


def test_min_scale_floor():
    r = ScaleRef(initial_scale_power=3, window=1000, hysteresis=1, min_scale=4.0)
    assert _run(r, [1, 1, 1]) == [4.0, 4.0, 4.0]
    assert r.skipped == 3 and r.step == 0


def test_clipping_multiplier():
    """mult = 1 / (S * max((||g|| / S + 1e-6) / max_norm, 1)), ||g|| the norm of the scaled gradients."""
    S = 1024.0
    for norm_unscaled, max_norm in ((3.0, 1.0), (0.25, 1.0), (7.5, 2.0)):
        r = ScaleRef(initial_scale_power=10, max_norm=max_norm)
        r.update((norm_unscaled * S) ** 2)
        want = 1.0 / (S * max((norm_unscaled + 1e-6) / max_norm, 1.0))
        assert math.isclose(float(r.grad_mult), want, rel_tol=1e-6)
        # the unscaled, clipped gradient has norm min(norm, ~max_norm)
        assert math.isclose(norm_unscaled * S * float(r.grad_mult), min(norm_unscaled, max_norm), rel_tol=1e-5)
    r = ScaleRef(initial_scale_power=10)  # clipping off: plain unscale
    r.update(1e6)
    assert float(r.grad_mult) == 1.0 / 1024.0


def test_clip_only_state_keeps_unit_scale():
    r = ScaleRef(dynamic=False, max_norm=1.0)
    r.update(16.0)
    assert float(r.scale) == 1.0 and math.isclose(float(r.grad_mult), 1.0 / (4.0 + 1e-6), rel_tol=1e-6)
    r.update(float("nan"))
    assert r.skip == 1 and r.skipped == 1 and float(r.scale) == 1.0 and r.step == 1
