"""CPU: the SD-VAE encode half and the latent extraction around it — the encode oracle against the unmodified
reference (tests/golden/make_golden_encode.py), the encoder module's parameter layout, the ADM centre crop, the
streaming LMDB writer, the ImageFolder order of extract_latent.py, and the GEMM plans the encoder's convolutions get."""
import os
import subprocess
import sys
import tracemalloc

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from maskdit_b200 import data as D  # noqa: E402

GOLD = os.path.join(ROOT, "tests", "golden")


def load(name):
    return {k: v for k, v in np.load(os.path.join(GOLD, name + ".npz")).items()}


def test_encode_oracle_matches_reference():
    """oracle/vae_encode_oracle.py vs FrozenAutoencoderKL.encode_moments / sample on the stand-in weights, B = 2 at
    64x64 (every layer type of the encoder: conv_in, ResnetBlocks with and without nin_shortcut, three stride-2
    Downsample convolutions, the AttnBlock, norm_out + conv_out, quant_conv), the mirrored images, and z."""
    from oracle import vae_encode_oracle as VE
    g = load("vae_encode")
    sd = VE.make_vae_encoder_state_dict(4)
    x = torch.from_numpy(g["x"])
    with torch.no_grad():
        m = VE.encode_moments(sd, x)
        mf = VE.encode_moments(sd, x.flip(-1))
    np.testing.assert_allclose(m.numpy(), g["moments"], rtol=1e-3, atol=2e-4)
    np.testing.assert_allclose(mf.numpy(), g["moments_flip"], rtol=1e-3, atol=2e-4)
    z = VE.sample(torch.from_numpy(g["moments"]), torch.from_numpy(g["eps"]))
    np.testing.assert_allclose(z.numpy(), g["z"], rtol=1e-6, atol=1e-7)
    assert 0 < g["bf16_rel_mean"] < 2e-2 and 0 < g["bf16_rel_logvar"] < 2e-2   # the yardstick the GPU bound uses


def test_stand_in_weights_leave_the_decoder_stand_in_alone():
    from oracle import vae_encode_oracle as VE
    from oracle import vae_oracle as VO
    a, b = VO.make_vae_state_dict(3), VO.make_vae_state_dict(3)
    VE.make_vae_encoder_state_dict(4)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    assert not set(VE.encoder_param_shapes()) & set(VO.decoder_param_shapes())


def test_encoder_parameter_counts_and_layout():
    from maskdit_b200.vae import AutoencoderKLEncoder
    sd = AutoencoderKLEncoder().state_dict()
    enc = {k: v for k, v in sd.items() if k.startswith("encoder.")}
    assert len(enc) == 106
    assert sum(v.numel() for v in enc.values()) == 34_163_592
    assert sum(v.numel() for k, v in sd.items() if k.startswith("quant_conv.")) == 72
    g = load("vae_encode")
    assert list(sd.keys()) == list(g["keys"])                          # the reference's keys in its order
    assert [str(tuple(v.shape)) for v in sd.values()] == list(g["shapes"])


def test_encoder_input_checks_and_fn_dispatch():
    from maskdit_b200.vae import AutoencoderKLEncoder
    e = AutoencoderKLEncoder()
    with pytest.raises(ValueError, match="multiples of 8"):
        e.encode_moments(torch.zeros(1, 3, 60, 64))
    with pytest.raises(ValueError):
        e.encode_moments(torch.zeros(1, 4, 64, 64))
    with pytest.raises(NotImplementedError):
        e(torch.zeros(1, 3, 64, 64), "decode")


def test_get_encoder_reads_the_encoder_half_of_a_checkpoint(tmp_path):
    from maskdit_b200.vae import get_encoder
    from oracle import vae_encode_oracle as VE
    from oracle import vae_oracle as VO
    enc = VE.make_vae_encoder_state_dict(4)
    torch.save({**enc, **VO.make_vae_state_dict(3)}, tmp_path / "full.pth")
    m = get_encoder(str(tmp_path / "full.pth"), device="cpu")
    sd = m.state_dict()
    assert sd.keys() == enc.keys() and all(torch.equal(sd[k], enc[k]) for k in enc)
    torch.save(VO.make_vae_state_dict(3), tmp_path / "decoder_only.pth")
    with pytest.raises(KeyError):
        get_encoder(str(tmp_path / "decoder_only.pth"), device="cpu")


def test_center_crop_matches_reference_bit_for_bit():
    from PIL import Image
    g = load("center_crop")
    for i in range(3):
        got = D.center_crop_arr(Image.fromarray(g[f"in{i}"]), 64)
        assert got.dtype == np.uint8 and np.array_equal(got, g[f"out{i}"]), i


def test_load_image_is_totensor_normalize(tmp_path):
    from PIL import Image
    rng = np.random.default_rng(3)
    arr = rng.integers(0, 256, (64, 64, 3), dtype=np.uint8)
    Image.fromarray(arr).save(tmp_path / "a.png")
    x = D.load_image(str(tmp_path / "a.png"), 64)
    want = (torch.from_numpy(arr).permute(2, 0, 1).float().div(255) - 0.5) / 0.5   # ToTensor + Normalize(0.5, 0.5)
    assert x.dtype == np.float32 and torch.equal(torch.from_numpy(x), want)


def test_mdb_writer_streams_large_values(tmp_path):
    """A few thousand 32 KB values (one 8x32x32 fp32 latent each) plus small values: everything reads back exactly, and
    the writer's peak Python allocation stays far below the bytes written."""
    n, vbytes = 3000, 32768
    path = str(tmp_path / "db")
    tracemalloc.start()
    with D.MdbWriter(path) as w:
        for i in range(n):
            w.put(f"z-{i}".encode(), np.random.default_rng(i).standard_normal(vbytes // 4).astype("<f4"))
            w.put(f"y-{i}".encode(), str(i % 1000).encode())
        w.put(b"length", str(n).encode())
    _, peak = tracemalloc.get_traced_memory()
    tracemalloc.stop()
    assert peak < n * vbytes / 20, peak                   # 98 MB written; the keys and page pointers are ~1 MB
    rd = D.MdbReader(path)
    assert rd.entries == 2 * n + 1 and bytes(rd.get(b"length")) == str(n).encode()
    for i in list(range(0, n, 97)) + [n - 1]:
        want = np.random.default_rng(i).standard_normal(vbytes // 4).astype("<f4").tobytes()
        assert bytes(rd.get(f"z-{i}".encode())) == want, i
        assert bytes(rd.get(f"y-{i}".encode())) == str(i % 1000).encode()
    assert rd.get(b"z-3000") is None
    rd.close()
    ds = D.ImageNetLatentDataset(str(tmp_path), resolution=32, split="db")
    z, onehot = ds[5]
    assert len(ds) == n and z.shape == (8, 32, 32) and onehot[5] == 1


def test_mdb_writer_rejects_duplicate_keys(tmp_path):
    w = D.MdbWriter(str(tmp_path / "db"))
    w.put(b"a", b"1")
    with pytest.raises(KeyError):
        w.put(b"a", b"2")
    w.put(b"b", bytes(5000))
    with pytest.raises(KeyError):
        w.put(b"b", bytes(5000))
    w.close()
    rd = D.MdbReader(str(tmp_path / "db"))
    assert bytes(rd.get(b"a")) == b"1" and bytes(rd.get(b"b")) == bytes(5000) and rd.entries == 2


def test_empty_mdb_writer(tmp_path):
    D.MdbWriter(str(tmp_path / "db")).close()
    rd = D.MdbReader(str(tmp_path / "db"))
    assert rd.entries == 0 and rd.get(b"x") is None


def test_image_folder_order_matches_torchvision(tmp_path):
    tvd = pytest.importorskip("torchvision.datasets")
    from PIL import Image
    root = tmp_path / "train"
    names = {"n02": ["b.JPEG", "a.png", "c.txt", "sub/z.jpg", "sub/a.bmp"], "n01": ["x.jpeg", "y.PNG"],
             "n10": ["0.webp"]}
    fmt = {"jpeg": "JPEG", "jpg": "JPEG", "png": "PNG", "bmp": "BMP", "webp": "WEBP"}
    for cls, files in names.items():
        for f in files:
            p = root / cls / f
            p.parent.mkdir(parents=True, exist_ok=True)
            if f.endswith(".txt"):
                p.write_text("not an image")
            else:
                Image.new("RGB", (4, 4)).save(p, format=fmt[f.rsplit(".", 1)[1].lower()])
    Image.new("RGB", (4, 4)).save(root / "loose.png")        # a file beside the class directories is not a class
    samples, classes = D.image_folder_samples(str(root))
    ref = tvd.ImageFolder(str(root))
    assert classes == ref.classes
    assert samples == [(p, y) for p, y in ref.imgs]


@pytest.mark.parametrize("res", [256, 512])
def test_encoder_convolutions_do_not_split_k(res):
    """The encoder's convolution GEMMs (store epilogue) run without k-slices at 256 and 512 px, so every output element
    is one fixed-order reduction: the moments are run-to-run and chunking invariant."""
    from maskdit_b200 import _lib
    from maskdit_b200.vae import AutoencoderKLEncoder
    shapes = set()
    H, cin = res, 4
    for k, shp in AutoencoderKLEncoder().state_dict().items():
        if not k.endswith(".weight") or len(shp) != 4 or k.startswith("quant_conv"):
            continue
        co, ci, kh, kw = shp
        if ".downsample." in k:
            H //= 2
        ci = 4 if k == "encoder.conv_in.weight" else ci
        Kp = (kh * kw * ci + 7) // 8 * 8
        M = H * H
        shapes.add((M, co, Kp))
        shapes.add((min(M * 64, 1 << 21), co, Kp))           # a batch of images per im2col operand
    T = (res // 8) ** 2
    shapes |= {(T, T, 512), (T, 512, T)}                     # the AttnBlock's q k^T and P v
    for M, N, K in sorted(shapes):
        plan = _lib.gemm_plan(M, N, K)
        assert plan["splits"] == 1, (M, N, K, plan)
    plan = _lib.gemm_plan(T, 512, T, b_mn=True)
    assert plan["splits"] == 1


def test_library_builds():
    r = subprocess.run([sys.executable, "-m", "maskdit_b200.build"], cwd=ROOT, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr[-2000:]
