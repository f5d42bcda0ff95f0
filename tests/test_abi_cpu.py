"""CPU-only checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/pika_b200.h declares (no compute calls without a GPU), and argument validation fails loudly."""
import ctypes
import json
import os
import re
import subprocess
import sys

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


# every long long query of the header with arguments a user can pass; the sizes from pk_rnnt_loss_workspace_bytes on grow with the
# batch and are above 2^32 here
LONG_LONG_QUERIES = {
    "pk_launch_count": (),
    "pk_colstats_ws_floats": (6000,),
    "pk_lstm_seq_workspace_bytes": (1024,),
    "pk_rnnt_loss_workspace_bytes": (4096, 1000, 200),
    "pk_rnnt_loss_colsum_workspace_bytes": (4096, 1000, 200, 6000),
    "pk_attention_keep_bits_bytes": (1024, 2048, 16),
    "pk_frontend_workspace_bytes": (4096, 160240, 1000, 80, 240),              # 4096 ten-second utterances: 9.2 GB
    "pk_frontend_noise_rir_workspace_bytes": (4096, 160240, 1000, 80, 240, 16000),
    "pk_conv_same_f64_workspace_bytes": (4096, 160240, 16000),
}

_CHILD_LONG_LONG = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from pika_b200 import _lib
out = {}
for name, args in json.loads(sys.stdin.read()).items():
    # the same symbol through a prototype of its own that returns long long, independent of the binding under test
    direct = ctypes.CFUNCTYPE(ctypes.c_longlong, *[ctypes.c_int] * len(args))((name, _lib.lib))
    out[name] = [getattr(_lib.lib, name)(*args), direct(*args)]
print(json.dumps(out))
"""


def test_long_long_queries_return_64_bit_values():
    """in a fresh interpreter (nothing else has touched the binding), each query returns the function's whole long long result"""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pika_b200.h")).read(), flags=re.S)
    declared = re.findall(r"\blong long\s+(pk_\w+)\s*\(", hdr)
    assert sorted(declared) == sorted(LONG_LONG_QUERIES)
    proc = subprocess.run([sys.executable, "-c", _CHILD_LONG_LONG, ROOT], input=json.dumps(LONG_LONG_QUERIES), capture_output=True,
                          text=True, timeout=300)
    assert proc.returncode == 0, proc.stderr
    res = json.loads(proc.stdout.strip().splitlines()[-1])
    assert list(res) == list(LONG_LONG_QUERIES)
    for i, (name, (got, full)) in enumerate(res.items()):
        assert got == full, "%s%s: %d, the function returned %d" % (name, LONG_LONG_QUERIES[name], got, full)
        assert i < 3 or full > 2 ** 32, name


_CHILD_REJECT = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from pika_b200 import _lib
A = 1 << 20
calls = [("pk_add", (A, A, A, 1, 64)),                       # no stream
         ("pk_add", (A, A, A, 1, 64, None, 0)),              # one argument too many
         ("pk_add", (A, A, A, 1.0, 64, None)),               # float for the int dtype
         ("pk_add", (A, A, A, 1, 64.0, None)),               # float for the long long element count
         ("pk_dropout", (A, A, 1, 64, 0.1, 1.5, None)),      # float for the uint32_t seed
         ("pk_gemm_bf16", (ctypes.byref(_lib.View4()), None))]   # another struct than pk_gemm_desc
out = []
for name, args in calls:
    before = _lib.launch_count()
    try:
        getattr(_lib.lib, name)(*args)
        raised = None
    except (TypeError, ctypes.ArgumentError) as e:
        raised = type(e).__name__
    out.append([name, raised, _lib.launch_count() - before])
print(json.dumps(out))
"""


def test_calls_that_disagree_with_the_header_raise_before_the_call():
    """a wrong argument count, a float for an integer parameter or the wrong struct raises in the binding and launches nothing.
    Run without a CUDA device and with made-up addresses, so that a call the binding let through could not run a kernel."""
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD_REJECT, ROOT], env=env, capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, proc.stderr
    res = json.loads(proc.stdout.strip().splitlines()[-1])
    assert len(res) == 6
    for i, (name, raised, launches) in enumerate(res):
        assert raised is not None, "call %d of %s went through" % (i, name)
        assert launches == 0


def header_structs():
    """{typedef name: [field names in order]} of the structs include/pika_b200.h declares"""
    hdr = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "pika_b200.h")).read(), flags=re.S)
    out = {}
    for body, name in re.findall(r"typedef\s+struct\s*\{(.*?)\}\s*(\w+)\s*;", hdr, flags=re.S):
        fields = []
        for decl in filter(str.strip, body.split(";")):
            first, *more = re.sub(r"\[[^\]]*\]", "", decl).split(",")     # "int a, b" declares a and b; drop array extents
            fields += [re.findall(r"\w+", first)[-1]] + [m.strip() for m in more]
        out[name] = fields
    return out


def test_struct_mirrors_match_the_c_layout(tmp_path):
    """sizeof and every field's offset and size, as the system C compiler lays the header's structs out, against the ctypes
    mirrors the binding passes"""
    from pika_b200 import _lib
    structs = header_structs()
    assert sorted(structs) == sorted(_lib.STRUCTS)
    lines = ["#include <stddef.h>", "#include <stdio.h>", '#include "pika_b200.h"', "int main(void) {"]
    for name, fields in structs.items():
        lines.append('printf("%s - %%zu %%zu\\n", (size_t)0, sizeof(%s));' % (name, name))
        lines += ['printf("%s %s %%zu %%zu\\n", offsetof(%s, %s), sizeof(((%s*)0)->%s));' % (name, f, name, f, name, f) for f in fields]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines + ["return 0;", "}"]) + "\n")
    exe = tmp_path / "layout"
    subprocess.run([os.environ.get("CC", "cc"), "-I", os.path.join(ROOT, "include"), "-o", str(exe), str(src)], check=True)
    c = {}
    for line in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.splitlines():
        name, field, off, size = line.split()
        c[name, field] = int(off), int(size)
    for name, fields in structs.items():
        mirror = _lib.STRUCTS[name]
        assert [f[0] for f in mirror._fields_] == fields, name
        assert ctypes.sizeof(mirror) == c[name, "-"][1], name
        for f in fields:
            assert (getattr(mirror, f).offset, getattr(mirror, f).size) == c[name, f], (name, f)


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
