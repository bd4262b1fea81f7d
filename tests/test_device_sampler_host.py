"""Host side of the on-device EOT draw (DorPatch.generate(eot_sampler="device")): a numpy restatement of the draw that
tests/test_gpu_device_sampler.py compares the kernel against bit for bit, its Philox4x32-10 against the published
known-answer vectors, the argument refusals that need no GPU, main.py's flag and the C ABI declarations."""
import os

import numpy as np
import pytest
import torch

from dorpatch_b200 import _lib
from dorpatch_b200.attack import DorPatch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
M32 = np.uint64(0xFFFFFFFF)


# ---- the restatement ------------------------------------------------------------------------------------------------
def philox4x32_10(c, k):
    """Philox4x32-10 of counters c (4 uint64 arrays holding 32-bit words) under key k (two ints)."""
    c0, c1, c2, c3 = (np.asarray(v, np.uint64) & M32 for v in c)
    k0, k1 = np.uint64(k[0]), np.uint64(k[1])
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c0
        p1 = np.uint64(0xCD9E8D57) * c2
        c0, c1, c2, c3 = ((p1 >> np.uint64(32)) ^ c1 ^ k0, p1 & M32, (p0 >> np.uint64(32)) ^ c3 ^ k1, p0 & M32)
        k0 = (k0 + np.uint64(0x9E3779B9)) & M32
        k1 = (k1 + np.uint64(0xBB67AE85)) & M32
    return c0, c1, c2, c3


def draw_below(key, pos, it, tag, n):
    """Uniform integers in [0, n) per position (Lemire's multiply-shift with rejection), as the kernel draws them."""
    pos = np.asarray(pos, np.uint64)
    n = np.asarray(n, np.uint64)
    out = np.zeros(pos.shape, np.int64)
    todo = np.ones(pos.shape, bool)
    reject = (np.uint64(2 ** 32) % n)
    attempt = 0
    while todo.any():
        words = philox4x32_10((pos, np.full_like(pos, it), np.full_like(pos, tag), np.full_like(pos, attempt)), key)
        for w in words:
            m = w * n
            ok = todo & ((m & M32) >= reject)
            out[ok] = (m >> np.uint64(32))[ok].astype(np.int64)
            todo &= ~ok
        attempt += 1
    return out


def sample_distinct(key, it, tag, n, m):
    """m distinct values of [0, n) in random order: Floyd's algorithm, then a Fisher-Yates shuffle."""
    s = np.arange(m)
    t = draw_below(key, s, it, tag, n - m + s + 1)
    u = draw_below(key, s, it, tag + (1 << 16), s + 1)
    seen, out = set(), []
    for j in range(m):
        v = int(t[j]) if int(t[j]) not in seen else n - m + j
        seen.add(v)
        out.append(v)
    for j in range(m - 1, 0, -1):
        out[j], out[int(u[j])] = out[int(u[j])], out[j]
    return np.asarray(out, np.int64)


def reference_draw(seed, stage, it, failed, n_mask, S, dual=False):
    """One image's draw: (idx [S], idx2 [S] or None, n_ff) for the failed set `failed` (indices) at step (stage, it)."""
    seed = int(seed) % 2 ** 64
    key = (seed & 0xFFFFFFFF, seed >> 32)
    members = np.asarray(sorted(int(v) for v in failed if v < n_mask), np.int64)
    n_ff = min(len(members), S // 2) if it >= 1000 else 0
    rows = []
    for d in range(2 if dual else 1):
        tag = stage | (d << 8)
        row = np.zeros(S, np.int64)
        if n_ff:
            row[:n_ff] = members[sample_distinct(key, it, tag, len(members), n_ff)]
        if S - n_ff:
            row[n_ff:] = sample_distinct(key, it, tag | (2 << 16), n_mask, S - n_ff)
        rows.append(row)
    return rows[0], (rows[1] if dual else None), n_ff


# ---- tests ----------------------------------------------------------------------------------------------------------
def test_philox_known_answers():
    """Random123's known-answer vectors for Philox4x32-10."""
    got = philox4x32_10(([0], [0], [0], [0]), (0, 0))
    assert [int(v[0]) for v in got] == [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]
    got = philox4x32_10(([0xFFFFFFFF], [0xFFFFFFFF], [0xFFFFFFFF], [0xFFFFFFFF]), (0xFFFFFFFF, 0xFFFFFFFF))
    assert [int(v[0]) for v in got] == [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]
    got = philox4x32_10(([0x243f6a88], [0x85a308d3], [0x13198a2e], [0x03707344]), (0xa4093822, 0x299f31d0))
    assert [int(v[0]) for v in got] == [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]


def test_reference_draw_semantics():
    """The restatement follows attack.py:193-218: n_ff, distinct parts, failed part inside the set."""
    failed = [3, 17, 40, 41, 99, 120]
    for it, want in ((999, 0), (1000, 6), (1500, 6)):
        idx, idx2, n_ff = reference_draw(7, 1, it, failed, 144, 32, dual=True)
        assert n_ff == want
        for row in (idx, idx2):
            assert set(row[:n_ff]) <= set(failed) and len(set(row[:n_ff])) == n_ff
            assert len(set(row[n_ff:])) == 32 - n_ff and row.min() >= 0 and row.max() < 144
    idx, _, n_ff = reference_draw(7, 1, 1000, list(range(0, 2520, 7)), 2520, 128)
    assert n_ff == 64                                     # min(|F|, S/2)
    assert not np.array_equal(reference_draw(7, 1, 1000, [], 144, 32)[0], reference_draw(8, 1, 1000, [], 144, 32)[0])
    assert not np.array_equal(reference_draw(7, 0, 1000, [], 144, 32)[0], reference_draw(7, 1, 1000, [], 144, 32)[0])
    assert np.array_equal(np.sort(reference_draw(3, 0, 5, [], 144, 144)[0]), np.arange(144))   # S = n_mask


def test_generate_refuses_bad_sampler(monkeypatch):
    x = torch.zeros(1, 3, 56, 56)
    with pytest.raises(ValueError, match="eot_sampler"):
        DorPatch().generate(None, x, 0.12, 1000, None, 0, eot_sampler="numpy")
    monkeypatch.setenv("DORPATCH_FAILED", "host")
    with pytest.raises(ValueError, match="DORPATCH_FAILED=host"):
        DorPatch().generate(None, x, 0.12, 1000, None, 0, eot_sampler="device")


def test_main_flag_and_result_path():
    from dorpatch_b200 import main as M
    from dorpatch_b200.utils import generate_saving_path
    args = M.parser.parse_args([])
    assert args.eot_sampler == "host"
    base = generate_saving_path(vars(args).copy())
    dev = generate_saving_path(vars(M.parser.parse_args(["--eot_sampler", "device"])).copy())
    assert "eot_sampler" not in base
    assert "__eot_sampler=device" in dev
    with pytest.raises(SystemExit):
        M.parser.parse_args(["--eot_sampler", "numpy"])


def test_abi_declares_the_sampler_entry_points():
    header = open(os.path.join(ROOT, "include", "dorpatch.h")).read()
    for name in ("dp_eot_universe_upload", "dp_eot_draw", "dp_eot_draw_rects", "dp_attack_grad_drawn",
                 "dp_failed_set_update_drawn"):
        assert "%s(" % name in header, name
        assert name in _lib.SIGNATURES, name
    assert _lib.ABI_VERSION == 9
