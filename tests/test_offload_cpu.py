"""CPU tier: AdamW state in host memory without a GPU — the placement of each parameter's state under a device budget
(`_state_placement`), the layout of the host block (`_host_layout`), the optimizer's argument checks, and the argument
checks of mm_adamw_host / mm_host_alloc / mm_host_free, which report errors before any CUDA call."""
import ctypes

import pytest
import torch


def _placement(numels, budget):
    from macaw_llm_b200.training import _state_placement

    return _state_placement(numels, budget)


def test_placement_none_is_all_device_and_zero_all_host():
    ns = [4096 * 4096, 7, 1, 32000 * 4096]
    assert _placement(ns, None) == [True] * 4
    assert _placement(ns, 0) == [False] * 4
    assert _placement([], 0) == [] and _placement([], None) == []


def test_placement_exact_fit_and_off_by_one():
    ns = [100, 50]
    assert _placement(ns, 12 * 150) == [True, True]
    assert _placement(ns, 12 * 150 - 1) == [True, False]
    assert _placement(ns, 12 * 100) == [True, False]
    assert _placement(ns, 12 * 100 - 1) == [False, True]  # the first no longer fits; the second still does
    assert _placement(ns, 12 * 50 - 1) == [False, False]


def test_placement_first_fit_skips_a_large_tensor():
    # the big one does not fit what is left after the first; the later small ones still go on the device
    ns = [10, 1000, 20, 30, 5]
    assert _placement(ns, 12 * 60) == [True, False, True, True, False]
    assert _placement(ns, 12 * 65) == [True, False, True, True, True]


def test_host_layout_aligned_and_exact():
    from macaw_llm_b200.training import _host_layout, _state_placement

    ns = [1, 7, 128, 4099, 3, 32, 5]
    place = _state_placement(ns, 12 * 20)
    assert place == [True, True, False, False, True, False, True]  # first-fit: 1, 7, 3 and 5 elements fit 20
    offs, total = _host_layout(ns, place)
    spans = []
    for n, p, o in zip(ns, place, offs):
        if p:
            assert o is None
            continue
        assert len(o) == 3 and all(x % 16 == 0 for x in o)
        for x in o:
            spans.append((x, x + 4 * n))
    spans.sort()
    assert all(a[1] <= b[0] for a, b in zip(spans, spans[1:]))  # no overlap
    want = sum(3 * ((4 * n + 15) // 16 * 16) for n, p in zip(ns, place) if not p)
    assert total == want and spans[-1][1] <= total < spans[-1][1] + 16
    assert _host_layout(ns, [True] * len(ns)) == ([None] * len(ns), 0)


def test_optimizer_rejects_bad_budgets_and_reports_host_bytes():
    from macaw_llm_b200.training import FusedAdamW

    ps = [torch.nn.Parameter(torch.zeros(10, 4)), torch.nn.Parameter(torch.zeros(3))]
    for bad in (-1, 1.5, True):
        with pytest.raises(ValueError, match="device_state_bytes"):
            FusedAdamW(ps, device_state_bytes=bad)
    assert FusedAdamW(ps).host_state_bytes == 0
    assert FusedAdamW(ps, device_state_bytes=12 * 40).host_state_bytes == 3 * 16
    assert FusedAdamW(ps, device_state_bytes=0).host_state_bytes == 3 * 160 + 3 * 16


def test_host_entries_report_errors_without_a_gpu():
    from macaw_llm_b200 import _lib

    lib = _lib.load()
    P = 1 << 20  # a fake, 16-byte aligned address: argument checks come before any CUDA call, nothing is dereferenced
    args = lambda **kw: [kw.get(k, d) for k, d in (("p", P), ("g", P), ("w", P), ("m", P), ("v", P), ("n", 16))]  # noqa: E731

    def call(**kw):
        return lib.mm_adamw_host(*args(**kw), 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None, 1.0, None, None, None)

    for k in ("p", "g", "w", "m", "v"):
        assert call(**{k: None}) != 0 and b"mm_adamw_host: bad arguments" in lib.mm_last_error(), k
    for n in (0, -5):
        assert call(n=n) != 0 and b"mm_adamw_host: bad arguments" in lib.mm_last_error(), n
    for k, off in (("w", 8), ("m", 4), ("v", 12), ("p", 2), ("g", 4)):
        assert call(**{k: P + off}) != 0 and b"mm_adamw_host: alignment" in lib.mm_last_error(), (k, off)
    # step 0 without a device step counter
    assert lib.mm_adamw_host(P, P, P, P, P, 16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 0, None, 1.0, None, None, None) != 0
    h, d = ctypes.c_void_p(), ctypes.c_void_p()
    for nbytes in (0, -1):
        assert lib.mm_host_alloc(nbytes, ctypes.byref(h), ctypes.byref(d)) != 0
        assert b"mm_host_alloc: bad arguments" in lib.mm_last_error()
    assert lib.mm_host_alloc(64, None, ctypes.byref(d)) != 0 and b"mm_host_alloc: bad arguments" in lib.mm_last_error()
    assert lib.mm_host_alloc(64, ctypes.byref(h), None) != 0 and b"mm_host_alloc: bad arguments" in lib.mm_last_error()
    assert lib.mm_host_free(None) != 0 and b"mm_host_free: null pointer" in lib.mm_last_error()
