"""CPU tier: the learning-rate schedule without a GPU — `LRSchedule.lr_lambda` against transformers' own lambdas (the
schedule HF Trainer hands DeepSpeed for train.sh's `--lr_scheduler_type cosine --warmup_ratio 0.03`), the warmup count
of a ratio against `TrainingArguments.get_warmup_steps`, the argument checks of `LRSchedule` / `FusedAdamW`, and the
argument checks of mm_lr_schedule, which report errors before any CUDA call."""
import ctypes
import functools
import types

import numpy as np
import pytest
import torch


def _hf_lambda(name, W, N):
    from transformers import optimization as O

    if name == "linear":
        return functools.partial(O._get_linear_schedule_with_warmup_lr_lambda, num_warmup_steps=W, num_training_steps=N)
    if name == "cosine":
        return functools.partial(O._get_cosine_schedule_with_warmup_lr_lambda, num_warmup_steps=W, num_training_steps=N,
                                 num_cycles=0.5)
    return functools.partial(O._get_constant_schedule_with_warmup_lr_lambda, num_warmup_steps=W)


@pytest.mark.parametrize("name", ["linear", "cosine", "constant_with_warmup"])
@pytest.mark.parametrize("N", [1, 10, 1000])
@pytest.mark.parametrize("W", [0, 1, 3, "N"])
def test_lr_lambda_equals_transformers(name, W, N):
    from macaw_llm_b200.training import LRSchedule

    W = N if W == "N" else W
    if W > N:
        with pytest.raises(ValueError, match="num_warmup_steps <= num_training_steps"):
            LRSchedule(name, W, N)
        return
    s, hf = LRSchedule(name, W, N), _hf_lambda(name, W, N)
    got = [s.lr_lambda(n) for n in range(N + 51)]
    want = [float(hf(n)) for n in range(N + 51)]
    assert got == want  # exactly: the same double arithmetic
    if name == "cosine" and N - W > 1:
        assert got[N + 1] > got[N]  # past N, HF's cosine rises again; not clamped


def test_lr_lambda_equals_lambdalr_over_a_dummy_optimizer():
    """The lr a LambdaLR from transformers.get_scheduler gives the optimizer at each step = fp32 of the restatement."""
    from transformers import get_scheduler

    from macaw_llm_b200.training import LRSchedule

    base, W, N = 3e-5, 3, 100
    for name in LRSchedule.NAMES:
        opt = torch.optim.SGD([torch.nn.Parameter(torch.zeros(1))], lr=base)
        sch = get_scheduler(name, opt, num_warmup_steps=W, num_training_steps=N)
        s = LRSchedule(name, W, N)
        for t in range(1, N + 20):  # the t-th update runs at the lr the scheduler set after t - 1 steps
            assert opt.param_groups[0]["lr"] == base * s.lr_lambda(t - 1), (name, t)
            assert s.lr_of_update(base, t) == float(np.float32(opt.param_groups[0]["lr"])), (name, t)
            opt.step()
            sch.step()


@pytest.mark.parametrize("ratio,N", [(0.03, 1000), (0.03, 10), (0.03, 100), (0.0, 50), (0.5, 7), (0.1, 30), (0.25, 3)])
def test_from_warmup_ratio_equals_training_arguments(ratio, N):
    from transformers import TrainingArguments

    from macaw_llm_b200.training import LRSchedule

    want = TrainingArguments.get_warmup_steps(types.SimpleNamespace(warmup_steps=ratio), N)
    s = LRSchedule.from_warmup_ratio("cosine", ratio, N)
    assert s.num_warmup_steps == want and s.num_training_steps == N
    assert LRSchedule.from_warmup_ratio("cosine", 0.03, 1000).num_warmup_steps == 30
    assert LRSchedule.from_warmup_ratio("cosine", 0.03, 10).num_warmup_steps == 1


def test_invalid_names_and_counts_raise():
    from macaw_llm_b200.training import FusedAdamW, LRSchedule

    for bad in ("cosine_with_restarts", "polynomial", "constant", "Cosine", ""):
        with pytest.raises(ValueError, match="supported: linear, cosine, constant_with_warmup"):
            LRSchedule(bad, 0, 10)
    for W, N in ((-1, 10), (0, 0), (11, 10), (1.5, 10), (0, 2.5), (True, 10), (0, 2 ** 31)):
        with pytest.raises(ValueError):
            LRSchedule("cosine", W, N)
    for r in (-0.01, 1.5, float("nan")):
        with pytest.raises(ValueError, match="warmup_ratio"):
            LRSchedule.from_warmup_ratio("cosine", r, 100)
    ps = [torch.nn.Parameter(torch.zeros(4))]
    with pytest.raises(TypeError, match="lr_schedule"):
        FusedAdamW(ps, lr_schedule="cosine")
    # without a schedule the lr is the base lr; with one, before any step, the first update's
    assert FusedAdamW(ps, lr=3e-5).last_lr() == 3e-5
    assert FusedAdamW(ps, lr=3e-5, lr_schedule=LRSchedule("cosine", 3, 100)).last_lr() == 0.0
    assert FusedAdamW(ps, lr=3e-5, lr_schedule=LRSchedule("cosine", 0, 100)).last_lr() == float(np.float32(3e-5))


def test_lr_schedule_entry_reports_errors_without_a_gpu():
    from macaw_llm_b200 import _lib

    lib = _lib.load()
    P = 1 << 20  # a fake address: argument checks come before any CUDA call, nothing is dereferenced

    def call(step=P, kind=1, W=3, N=100, out=P):
        return lib.mm_lr_schedule(step, 3e-5, kind, W, N, out, None)

    assert call(step=None) != 0 and b"mm_lr_schedule: bad arguments" in lib.mm_last_error()
    assert call(out=None) != 0 and b"mm_lr_schedule: bad arguments" in lib.mm_last_error()
    for kind in (-1, 3, 7):
        assert call(kind=kind) != 0 and b"mm_lr_schedule: unknown kind" in lib.mm_last_error(), kind
    for W, N in ((-1, 100), (0, 0), (0, -3), (101, 100)):
        assert call(W=W, N=N) != 0 and b"mm_lr_schedule: bad step counts" in lib.mm_last_error(), (W, N)


def test_adamw_entries_take_lr_dev_and_keep_the_abi5_argument_list():
    """lr_dev sits between skip_dev and stream in mm_adamw / mm_adamw_host.  A Python call written against ABI 5 (17
    arguments, without it) still binds: its 17th argument still arrives as `stream` and lr_dev as NULL.  Checked on a
    fake entry with the real argument types, which records what it receives, and on the bound library entries."""
    from macaw_llm_b200 import _lib

    class Fake:
        def __init__(self, argtypes):
            self.argtypes, self.got = argtypes, None

        def __call__(self, *args):
            self.got = args
            return 0

    stream, lr_dev = 0x7F00DEADBEEF, 0x7F00CAFE0000
    abi5 = (1, 2, 3, 4, 5, 16, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, 6, 1.0, 7, 8)  # every argument before lr_dev / stream
    for name in ("mm_adamw", "mm_adamw_host"):
        argtypes = _lib.SIGNATURES[name][1]
        assert len(argtypes) == 18 and argtypes[16] is ctypes.c_void_p and argtypes[17] is ctypes.c_void_p, name
        fake = Fake(argtypes)
        wrapped = _lib._NullableBeforeStream(fake, _lib.NULLABLE_BEFORE_STREAM[name])
        wrapped(*abi5, stream)  # ABI 5: 17 arguments, the stream last
        assert fake.got == abi5 + (None, stream), name
        wrapped(*abi5, lr_dev, stream)  # ABI 6: all 18, passed through unchanged
        assert fake.got == abi5 + (lr_dev, stream), name
        for short in (abi5[:-1] + (stream,), abi5 + (lr_dev, stream, 9)):  # any other count reaches ctypes unchanged
            wrapped(*short)
            assert fake.got == short, name

    lib = _lib.load()
    assert _lib.ABI_VERSION == 8 and lib.mm_abi_version() == 8
    for name in ("mm_adamw", "mm_adamw_host"):
        fn = getattr(lib, name)
        assert isinstance(fn, _lib._NullableBeforeStream) and len(fn.argtypes) == 18, name
        # n = 0: refused by the argument check, with and without lr_dev
        P = 1 << 20
        assert fn(P, P, P, P, P, 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None, 1.0, None, None, P, None) != 0
        assert fn(P, P, P, P, P, 0, 1e-3, 0.9, 0.999, 1e-8, 0.0, 1, None, 1.0, None, None, None) != 0
        assert b"bad arguments" in lib.mm_last_error()
