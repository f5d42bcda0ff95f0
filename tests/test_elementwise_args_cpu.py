"""Argument rejection of the memory-bound entry points of csrc/elementwise.cu: misaligned 16-byte vector operands, C % 8 != 0,
LayerNorm C > 1024, rows == 0, a drop probability of 0.  And of the persistent LSTM recurrence (csrc/lstm_seq.cu,
pk_lstm_seq_fwd_ex / _bwd_ex): a w_hh, workspace or dG that is not 16-byte aligned (16-byte loads and cp.async.bulk sources),
B == 0, U == 0, n_dir == 3, H % 64 != 0, n_dir * H/8 above the SM count, ldo < n_dir * H.  Each rejected call must return < 0 with
a pk_last_error message naming the problem, and launch nothing.

The calls run in a subprocess that sees no CUDA device (CUDA_VISIBLE_DEVICES=""), with made-up device addresses: should a check
regress, the call gets as far as a launch and fails with "no device" rather than the expected message, instead of running a kernel on
a bogus pointer.  With no device the SM count the LSTM check compares against is the H100's 132."""
import json
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

A, M = 1 << 20, (1 << 20) + 4               # a 16-byte aligned address and one that is only 4-byte aligned
F32, BF16 = 0, 1

# (id, expected message fragment, entry point, arguments); arguments are ("p", address) | ("L" | "I" | "F" | "U", value)
P = lambda a: ("p", a)
L = lambda v: ("L", v)
I = lambda v: ("I", v)
F = lambda v: ("F", v)
U = lambda v: ("U", v)


def _bn_fwd(x=A, y=A, C=256, rows=64, train=1, ws=A, dtype=F32):
    return ("pk_bn_fwd", P(x), P(y), I(dtype), L(rows), I(C), P(A), P(A), F(1e-5), I(train), F(0.1), P(A), P(A), P(A), P(A), P(ws))


def _bn_bwd(dy=A, x=A, dx=A, C=256, rows=64, ws=A):
    return ("pk_bn_bwd", P(dy), P(x), P(dx), I(BF16), L(rows), I(C), P(A), P(A), P(A), I(1), I(1), P(A), P(A), P(ws))


def _colsum(x=A, C=256, rows=64, ws=A):
    return ("pk_colsum", P(x), I(F32), L(rows), I(C), P(A), P(ws))


def _ln_fwd(x=A, y=A, C=256, rows=64):
    return ("pk_layernorm_fwd", P(x), P(y), I(BF16), L(rows), I(C), P(A), P(A), F(1e-6), P(A), P(A))


def _ln_bwd(dy=A, x=A, dx=A, C=256, rows=64):
    return ("pk_layernorm_bwd", P(dy), P(x), P(dx), I(F32), L(rows), I(C), P(A), P(A), P(A), P(A), P(A))


def _gather(src=A, dst=A, C=256, rows=64):
    return ("pk_gather_rows", P(src), P(A), P(dst), I(BF16), L(rows), I(C))


def _lstm_fwd(w_hh=A, ws=A, B=32, U=10, H=256, n_dir=1, ldo=None):
    ldo = n_dir * H if ldo is None else ldo
    return ("pk_lstm_seq_fwd_ex", P(A), P(w_hh), P(A), I(BF16), I(ldo), P(A), P(A), P(0), I(B), I(U), I(H), I(n_dir), I(0), P(ws))


def _lstm_bwd(dG=A, ws=A, B=32, U=10, H=256, n_dir=1, ldo=None):
    ldo = n_dir * H if ldo is None else ldo
    return ("pk_lstm_seq_bwd_ex", P(A), I(BF16), I(ldo), P(A), P(A), P(A), P(dG), P(0), I(B), I(U), I(H), I(n_dir), I(0), P(ws))


ALIGN = "16-byte aligned"
SMS = "#SMs"
CASES = [
    ("bn_fwd-x", ALIGN, _bn_fwd(x=M)),
    ("bn_fwd-y", ALIGN, _bn_fwd(y=M, dtype=BF16)),
    ("bn_fwd-ws", ALIGN, _bn_fwd(ws=M)),
    ("bn_fwd-C%8", "multiple of 8", _bn_fwd(C=252)),
    ("bn_fwd-rows0", "rows > 0", _bn_fwd(rows=0)),
    ("bn_fwd-eval-rows0", "rows > 0", _bn_fwd(rows=0, train=0)),
    ("bn_bwd-dy", ALIGN, _bn_bwd(dy=M)),
    ("bn_bwd-x", ALIGN, _bn_bwd(x=M)),
    ("bn_bwd-dx", ALIGN, _bn_bwd(dx=M)),
    ("bn_bwd-ws", ALIGN, _bn_bwd(ws=M)),
    ("bn_bwd-C%8", "multiple of 8", _bn_bwd(C=12)),
    ("bn_bwd-rows0", "rows > 0", _bn_bwd(rows=0)),
    ("colsum-x", ALIGN, _colsum(x=M)),
    ("colsum-ws", ALIGN, _colsum(ws=M)),
    ("colsum-C%8", "multiple of 8", _colsum(C=6004)),
    ("colsum-rows0", "rows > 0", _colsum(rows=0)),
    ("ln_fwd-x", ALIGN, _ln_fwd(x=M)),
    ("ln_fwd-y", ALIGN, _ln_fwd(y=M)),
    ("ln_fwd-C1032", "<= 1024", _ln_fwd(C=1032)),
    ("ln_fwd-C%8", "multiple of 8", _ln_fwd(C=260)),
    ("ln_fwd-rows0", "rows > 0", _ln_fwd(rows=0)),
    ("ln_bwd-dy", ALIGN, _ln_bwd(dy=M)),
    ("ln_bwd-x", ALIGN, _ln_bwd(x=M)),
    ("ln_bwd-dx", ALIGN, _ln_bwd(dx=M)),
    ("ln_bwd-C1032", "<= 1024", _ln_bwd(C=1032)),
    ("ln_bwd-rows0", "rows > 0", _ln_bwd(rows=0)),
    ("gather_rows-src", ALIGN, _gather(src=M)),
    ("gather_rows-dst", ALIGN, _gather(dst=M)),
    ("gather_rows-C%8", "multiple of 8", _gather(C=1030)),
    ("dropout-x", ALIGN, ("pk_dropout", P(M), P(A), I(F32), L(64), F(0.1), U(1))),
    ("dropout-p0", "p must be > 0", ("pk_dropout", P(A), P(A), I(F32), L(64), F(0.0), U(1))),
    ("mask_nz-dx", ALIGN, ("pk_mask_nz", P(A), P(A), P(M), I(BF16), L(64), F(1.0))),
    ("add-b", ALIGN, ("pk_add", P(A), P(M), P(A), I(BF16), L(64))),
    ("scatter_add_rows-rows0", "rows must be > 0", ("pk_scatter_add_rows", P(A), P(A), P(A), I(F32), L(0), I(13))),
    ("ce_grad-n>ld", "bad shape", ("pk_ce_grad", P(A), I(F32), L(32), P(A), P(A), F(1.0), P(A), L(4), I(33))),
    ("cast_split-cols_pad<cols", "bad shape", ("pk_cast_split", P(A), I(F32), L(64), P(A), P(A), L(64), L(4), I(64), I(56), F(1.0))),
    ("lstm_fwd-w_hh", ALIGN, _lstm_fwd(w_hh=M)),
    ("lstm_fwd-ws", ALIGN, _lstm_fwd(ws=M)),
    ("lstm_fwd-B0", "empty batch", _lstm_fwd(B=0)),
    ("lstm_fwd-U0", "U must be >= 1", _lstm_fwd(U=0)),
    ("lstm_fwd-n_dir3", "n_dir must be 1 or 2", _lstm_fwd(n_dir=3)),
    ("lstm_fwd-H%64", "multiple of 64", _lstm_fwd(H=200)),
    ("lstm_fwd-H1088", SMS, _lstm_fwd(H=1088)),
    ("lstm_fwd-bidir-H576", SMS, _lstm_fwd(H=576, n_dir=2)),
    ("lstm_fwd-ldo<n_dir*H", "ldo must be >= n_dir * H", _lstm_fwd(H=256, n_dir=2, ldo=504)),
    ("lstm_bwd-dG", ALIGN, _lstm_bwd(dG=M)),
    ("lstm_bwd-ws", ALIGN, _lstm_bwd(ws=M)),
    ("lstm_bwd-B0", "empty batch", _lstm_bwd(B=0)),
    ("lstm_bwd-U0", "U must be >= 1", _lstm_bwd(U=0)),
    ("lstm_bwd-n_dir3", "n_dir must be 1 or 2", _lstm_bwd(n_dir=3)),
    ("lstm_bwd-H%64", "multiple of 64", _lstm_bwd(H=200)),
    ("lstm_bwd-H1088", SMS, _lstm_bwd(H=1088)),
    ("lstm_bwd-bidir-H576", SMS, _lstm_bwd(H=576, n_dir=2)),
    ("lstm_bwd-ldo<n_dir*H", "ldo must be >= n_dir * H", _lstm_bwd(H=512, ldo=448)),
]

_CHILD = r"""
import ctypes, json, sys
sys.path.insert(0, sys.argv[1])
from pika_b200 import _lib
T = {"p": ctypes.c_void_p, "L": ctypes.c_longlong, "I": ctypes.c_int, "F": ctypes.c_float, "U": ctypes.c_uint32}
out = []
for name, *args in json.loads(sys.stdin.read()):
    before = _lib.launch_count()
    rc = getattr(_lib.lib, name)(*[T[k](v) for k, v in args], ctypes.c_void_p(0))
    out.append([rc, _lib.lib.pk_last_error().decode(), _lib.launch_count() - before])
print(json.dumps(out))
"""


@pytest.fixture(scope="module")
def results():
    env = dict(os.environ, CUDA_VISIBLE_DEVICES="")
    proc = subprocess.run([sys.executable, "-c", _CHILD, ROOT], input=json.dumps([c[2] for c in CASES]), env=env,
                          capture_output=True, text=True, timeout=300)
    assert proc.returncode == 0, proc.stderr
    res = json.loads(proc.stdout.strip().splitlines()[-1])
    assert len(res) == len(CASES)
    return res


@pytest.mark.parametrize("case", range(len(CASES)), ids=[c[0] for c in CASES])
def test_rejects_bad_arguments(results, case):
    cid, msg, (name, *_) = CASES[case]
    rc, err, launches = results[case]
    assert rc < 0, "%s (%s) accepted bad arguments (rc=%d, %r)" % (name, cid, rc, err)
    assert msg in err, "%s (%s): expected %r in %r" % (name, cid, msg, err)
    assert launches == 0
