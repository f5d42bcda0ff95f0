"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/pika_b200.h declares (no compute calls without a GPU), and argument validation fails loudly."""
import ctypes
import os
import re

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "pika_b200.h")).read()
    hdr = re.sub(r"/\*.*?\*/", "", hdr, flags=re.S)
    return sorted(set(re.findall(r"\b(pk_[a-z0-9_]+)\s*\(", hdr)))


def test_library_exports_every_declared_symbol():
    from pika_b200 import _lib
    syms = declared_symbols()
    assert len(syms) >= 35
    missing = [s for s in syms if not hasattr(_lib.lib, s)]
    assert not missing, missing
    assert _lib.lib.pk_version() >= 100
    assert isinstance(_lib.launch_count(), int)


def test_gemm_descriptor_validation_fails_loudly():
    from pika_b200 import _lib
    d = _lib.GemmDesc()
    d.n_pairs = 0
    rc = _lib.lib.pk_gemm_bf16(ctypes.byref(d), None)
    assert rc != 0 and b"n_pairs" in _lib.lib.pk_last_error()
    with pytest.raises(_lib.PikaError):
        _lib.check(rc, "pk_gemm_bf16")


def test_workspace_queries_are_pure_host_functions():
    from pika_b200 import _lib
    assert _lib.lib.pk_rnnt_loss_workspace_bytes(32, 240, 151) > 32 * 240 * 151 * 12
    _lib.lib.pk_frontend_workspace_bytes.restype = ctypes.c_longlong
    assert _lib.lib.pk_frontend_workspace_bytes(32, 160240, 1000, 80, 240) > 32 * 160240 * 12
    # row pitch of the fused attention's lse / D vectors: T rounded up to 64
    assert [_lib.lib.pk_attention_lse_stride(T) for T in (1, 63, 64, 65, 1000, 2048)] == [64, 64, 64, 128, 1024, 2048]


def test_softmax_bwd_rejects_bad_shapes_before_touching_the_device():
    """pk_softmax_bwd validates what its forward validates: n <= ld_p, ld_d >= ld_p, rows > 0"""
    import ctypes as C
    from pika_b200 import _lib
    L, I, F, U, NULL = C.c_longlong, C.c_int, C.c_float, C.c_uint32, C.c_void_p(0)
    for ld_d, ld_p, rows, n in ((64, 64, 16, 72), (56, 64, 16, 64), (64, 64, 0, 64), (64, 64, 16, 0)):
        rc = _lib.lib.pk_softmax_bwd(NULL, L(ld_d), NULL, L(ld_p), NULL, I(0), L(rows), I(n), F(0.0), U(0), NULL)
        assert rc < 0 and b"softmax rows" in _lib.lib.pk_last_error()


def test_no_product_module_imports_the_oracle():
    """oracle/ is test infrastructure: nothing under pika_b200/ may import it."""
    bad = []
    for dirpath, _, files in os.walk(os.path.join(ROOT, "pika_b200")):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dirpath, f)).read()
                if re.search(r"^\s*(from|import)\s+oracle\b", src, flags=re.M):
                    bad.append(os.path.join(dirpath, f))
    assert not bad, bad


def test_specaugment_draws_match_reference_streams(golden_dir):
    """utils/spec_augment.py parity: identical masks from identically seeded torch + numpy RNG streams."""
    import numpy as np
    import torch
    from pika_b200.utils.spec_augment import SpecAugment
    d = np.load(os.path.join(golden_dir, "specaug.npz"))
    for i in range(4):
        seed = int(d["seed_%d" % i])
        torch.manual_seed(seed)
        np.random.seed(seed)
        x = torch.ones(3, 200, 240)
        sa = SpecAugment(15, 35)
        sa.apply(x)
        sa.apply(x)
        np.testing.assert_array_equal(np.packbits((x[0] == 0).numpy()), d["mask_%d" % i])


def test_frontend_length_arithmetic_and_fbank_config(tmp_path):
    from pika_b200.frontend import FbankOptions, Frontend
    new_len, frames = Frontend.lengths([160240, 32240, 399, 1000], [1.0, 0.9, 1.0, 1.1])
    assert new_len == [160240, int(32240 / 0.9), 399, int(1000 / 1.1)]
    assert frames == [1000, 1 + (int(32240 / 0.9) - 400) // 160, 0, 1 + (909 - 400) // 160]
    cfg = tmp_path / "fbank.conf"
    cfg.write_text("--window-type=hamming \n--sample-frequency=16000\n--dither=1\n--low-freq=40    # low cutoff\n"
                   "--high-freq=-200 # relative to Nyquist\n--num-mel-bins=80\n")
    o = FbankOptions.from_config(str(cfg))
    assert (o.window_type, o.num_mel_bins, o.low_freq, o.high_freq, o.dither) == ("hamming", 80, 40.0, -200.0, 1.0)
    bad = tmp_path / "bad.conf"
    bad.write_text("--use-energy=true\n")
    with pytest.raises(ValueError):
        FbankOptions.from_config(str(bad))
