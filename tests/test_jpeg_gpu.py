"""GPU tier of the device JPEG decoder (mm_jpeg_decode): every supported file of tests/golden/jpeg.npz decodes to Pillow's
pixels bit for bit, batching and repetition change nothing, decode -> image() reproduces the reference's `_transform(224)`,
get_self_inputs takes JPEG bytes and paths, and corrupt scan bytes come back as ValueError from the status word.
No Pillow here: expected values are the stored fixtures and tests/jpeg_ref.py."""
import hashlib

import numpy as np
import pytest
import torch

from tests import jpeg_ref
from tests.golden.make_jpeg_golden import TF_ROWS
from tests.test_jpeg_cpu import MEAN_STD, NAMES, Z, corrupt, fixture, pil_matches

SUPPORTED = [(k, n["name"]) for k, n in enumerate(NAMES) if n["outcome"] == "ok"]


def _pipe(**kw):
    from macaw_llm_b200.inputs import DeviceInputPipeline

    return DeviceInputPipeline("cuda", torch.bfloat16, **kw)


@pytest.mark.gpu
def test_every_supported_file_decodes_bit_exactly():
    pipe = _pipe()
    out = pipe.decode_jpegs([Z[f"f{k}_jpeg"].tobytes() for k, _ in SUPPORTED])
    for (k, name), t in zip(SUPPORTED, out):
        assert t.is_cuda and t.dtype == torch.uint8 and t.shape == (NAMES[k]["h"], NAMES[k]["w"], 3), name
        assert pil_matches(k, t.cpu().numpy()), name


@pytest.mark.gpu
def test_mixed_batch_equals_single_decodes_and_runs_repeat():
    pipe = _pipe()
    items = [Z[f"f{k}_jpeg"].tobytes() for k, _ in SUPPORTED[::-1]]
    batch = [t.cpu() for t in pipe.decode_jpegs(items)]
    again = [t.cpu() for t in pipe.decode_jpegs(items)]
    for b, a, it in zip(batch, again, items):
        assert torch.equal(b, a)
        assert torch.equal(b, pipe.decode_jpegs([it])[0].cpu())


@pytest.mark.gpu
def test_decode_then_image_equals_reference_transform():
    pipe = _pipe()
    mean, std = MEAN_STD
    for tag in ("color", "gray"):
        k = int(Z[f"tf_{tag}_file"])
        out32, u8 = pipe.image(Z[f"f{k}_jpeg"].tobytes(), want_u8=True, fp32=True)
        crop = u8.cpu().numpy()
        assert hashlib.sha256(crop.tobytes()).digest() == Z[f"tf_{tag}_u8_sha"].tobytes(), tag
        assert np.array_equal(crop[TF_ROWS], Z[f"tf_{tag}_u8_rows"]), tag
        want = ((crop.astype(np.float32) / 255.0).transpose(2, 0, 1) - mean[:, None, None]) / std[:, None, None]
        got = out32.cpu().numpy()
        assert np.abs(got - want).max() < 1e-6, tag
        assert np.abs(got[:, TF_ROWS] - Z[f"tf_{tag}_f32_rows"]).max() < 1e-6, tag   # torchvision's own tensor


@pytest.mark.gpu
def test_get_self_inputs_with_bytes_and_paths(tmp_path):
    pipe = _pipe(n_frames=3)
    names = ["s300x400_q75_sub1", "s224_q90_gray_rst_rows2", "s479x641_q75_sub2_rst_rows1", "s224_q75_sub0_opt",
             "s33x65_q75_sub2"]
    raw = [fixture(n)[1] for n in names]
    paths = []
    for n, r in zip(names, raw):
        p = tmp_path / f"{n}.jpg"
        p.write_bytes(r)
        paths.append(p)
    arrays = [torch.from_numpy(jpeg_ref.decode(r)) for r in raw]
    ids = torch.randint(3, 500, (2, 8))
    batch = dict(input_ids=ids, attention_mask=torch.ones(2, 8, dtype=torch.int64), labels=ids.clone())
    auds = [None, None]

    def run(m):
        return pipe.get_self_inputs(batch, [m[0], None], auds, [None, [m[2], m[3], m[4]]])["inputs"]

    want = run(arrays)
    for got in (run(raw), run([str(p) for p in paths]), run(paths)):
        assert set(got) == set(want)
        for key, v in want.items():
            assert (v is None and got[key] is None) or torch.equal(got[key], v), key
    imgs = pipe.images([raw[1], None, arrays[0]])
    assert torch.equal(imgs[0], pipe.images([arrays[1]])[0]) and float(imgs[1].abs().max()) == 0
    assert torch.equal(imgs[2], want["images"][0])


@pytest.mark.gpu
def test_corrupt_scan_raises_value_error_from_the_status_word():
    pipe = _pipe()
    good = fixture("s224_q75_sub1_rst_blocks1")[1]
    for name in ("s224_q95_sub2", "s300x400_q75_sub1"):
        with pytest.raises(ValueError, match=r"<bytes #1>: corrupt JPEG data"):
            pipe.decode_jpegs([good, corrupt(fixture(name)[1])])
    # the decoder is still usable afterwards
    assert pil_matches(fixture("s224_q75_sub1_rst_blocks1")[0], pipe.decode_jpegs([good])[0].cpu().numpy())
