"""Device image pre-processing (csrc/preprocess.cu through the C ABI) against the Pillow/HF golden vectors and
oracle/clip_preprocess_oracle.py: integer work, so the bar is bit-exact (float32 result identical; f16/bf16 = the
round-to-nearest cast of it).

The per-thread code of both kernels is also replayed on the host bit for bit by tests/test_preprocess_core_cpu.py; these tests
are ordinary tests: a mismatch fails the suite."""
import hashlib
import os

import numpy as np
import pytest
import torch

import clip_preprocess_oracle as P

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
pytestmark = pytest.mark.gpu


def sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


@pytest.fixture(scope="module")
def proc():
    from visualcla.image_processing_vcla import VclaImageProcessor
    return VclaImageProcessor()


def test_golden_cases_bit_exact(proc):
    gold = np.load(os.path.join(ROOT, "tests", "golden", "preprocess.npz"))
    for i, (h, w) in enumerate(gold["cases"].tolist()):
        img = P.synthetic_image(h, w, seed=3 * h + w)
        px = proc(img).pixel_values
        assert px.shape == (1, 3, 224, 224) and px.dtype == torch.float32 and px.is_cuda
        assert sha(px[0].cpu().numpy()) == str(gold[f"px_sha_{i}"]), f"pixel_values differ from CLIPImageProcessor for {h}x{w}"


def test_random_shapes_vs_oracle(proc):
    rng = np.random.default_rng(21)
    shapes = [(1, 1), (2, 3), (224, 1), (1, 224), (223, 225), (449, 447), (31, 1500), (1500, 31), (1080, 1920), (3000, 2000)]
    shapes += [(int(rng.integers(2, 900)), int(rng.integers(2, 900))) for _ in range(10)]
    for h, w in shapes:
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        got = proc(img).pixel_values[0].cpu().numpy()
        assert np.array_equal(got, P.clip_preprocess(img)), (h, w)


def test_batch_list_pil_and_device_input(proc):
    from PIL import Image
    rng = np.random.default_rng(3)
    imgs = [rng.integers(0, 256, size=s + (3,), dtype=np.uint8) for s in [(300, 200), (64, 640), (224, 224)]]
    want = np.stack([P.clip_preprocess(a) for a in imgs])
    got = proc([Image.fromarray(imgs[0]), imgs[1], torch.from_numpy(imgs[2]).cuda()]).pixel_values
    assert np.array_equal(got.cpu().numpy(), want)
    # a palette / RGBA picture goes through PIL's convert("RGB") like HF's do_convert_rgb
    rgba = Image.fromarray(np.dstack([imgs[0], np.full(imgs[0].shape[:2], 77, np.uint8)]))
    assert np.array_equal(proc(rgba).pixel_values[0].cpu().numpy(), P.clip_preprocess(np.asarray(rgba.convert("RGB"))))


def test_half_and_bf16_are_rounded_casts():
    from visualcla.image_processing_vcla import VclaImageProcessor
    img = P.synthetic_image(333, 500, seed=9)
    want = torch.from_numpy(P.clip_preprocess(img))
    for dt in (torch.float16, torch.bfloat16):
        got = VclaImageProcessor(dtype=dt)(img).pixel_values[0].cpu()
        assert got.dtype == dt and torch.equal(got, want.to(dt))


def test_small_side_of_the_tiny_config():
    from visualcla.image_processing_vcla import VclaImageProcessor
    p56 = VclaImageProcessor(size={"shortest_edge": 56}, crop_size={"height": 56, "width": 56})
    rng = np.random.default_rng(8)
    for h, w in [(100, 80), (56, 56), (30, 200)]:
        img = rng.integers(0, 256, size=(h, w, 3), dtype=np.uint8)
        assert np.array_equal(p56(img).pixel_values[0].cpu().numpy(), P.clip_preprocess(img, 56))


def test_feeds_the_vision_tower(proc):
    """The result is accepted by the engine exactly like the HF processor's tensor (same values -> same embeddings)."""
    import visualcla
    from visualcla.engine import path_config_7b
    cfg = dict(path_config_7b(), v_layers=1, r_layers=1, t_hidden=256, t_heads=2, t_ffn=448, t_layers=1, t_vocab=1003)
    m = visualcla.VisualCLAModel.from_synthetic(cfg, seed=1, max_batch=2, max_seq=160)
    img = P.synthetic_image(480, 640, seed=4)
    dev = proc(img).pixel_values
    host = torch.from_numpy(P.clip_preprocess(img))[None].cuda()
    assert torch.equal(m.embed_images(dev), m.embed_images(host))


def test_errors_are_loud(proc):
    from visualcla import _native as N
    with pytest.raises(ValueError):
        proc(np.zeros((10, 10), np.uint8))                 # not RGB
    with pytest.raises(ValueError):
        proc(np.zeros((10, 10, 3), np.float32))            # not bytes
    with pytest.raises(N.NativeError):
        proc(np.zeros((1, 40000, 3), np.uint8))            # beyond the supported picture size
