"""The key encodings of the device key sort (tuplex_b200/csrc/keyhash.cuh sort_key_i64 / sort_str_word / sort_str_class), built for
the CPU through tests/sort_host.cpp, ordered as Python orders the keys: i64 as ints, strings as bytes (and, for valid UTF-8, as str),
also when a tied group of strings skips the words all its members share with its first member."""
import ctypes as ct
import os
import random
import subprocess

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))


@pytest.fixture(scope="module")
def host(tmp_path_factory):
    so = str(tmp_path_factory.mktemp("sort_host") / "sort_host.so")
    subprocess.check_call(["g++", "-O1", "-x", "c++", "-std=c++17", "-fPIC", "-shared", "-o", so, os.path.join(HERE, "sort_host.cpp")])
    L = ct.CDLL(so)
    L.h_sort_key_i64.argtypes, L.h_sort_key_i64.restype = [ct.c_longlong], ct.c_ulonglong
    L.h_sort_str_word.argtypes, L.h_sort_str_word.restype = [ct.c_char_p, ct.c_uint, ct.c_uint], ct.c_ulonglong
    L.h_sort_str_class.argtypes, L.h_sort_str_class.restype = [ct.c_uint, ct.c_uint], ct.c_uint
    return L


def _seq(L, b: bytes, k0: int = 0):
    """(word_k, class_k) from word k0 up to the first class below 9: what the string refinement compares, round after round."""
    out, k = [], k0
    while True:
        c = L.h_sort_str_class(len(b), k)
        out.append((L.h_sort_str_word(b, len(b), k), c))
        if c < 9:
            return out
        k += 1


def _shared_words(L, b: bytes, f: bytes, k: int) -> int:
    """sort_lcp_kernel's rule: words from k on that b shares with f, both with class 9."""
    w = 0
    while (L.h_sort_str_class(len(b), k + w) == 9 and L.h_sort_str_class(len(f), k + w) == 9
           and L.h_sort_str_word(b, len(b), k + w) == L.h_sort_str_word(f, len(f), k + w)):
        w += 1
    return w


def _strings(rng: random.Random):
    alpha = [0, 1, 0x41, 0x61, 0x7F, 0x80, 0xC3, 0xFE, 0xFF]
    out = [b"", b"\0", b"\0\0", b"a", b"a\0", b"a\0\0", b"ab", b"\xff", b"\xff\xff"]
    for n in range(41):  # every length 0-40, so every multiple of 8 and its neighbours
        for _ in range(6):
            out.append(bytes(rng.choice(alpha) for _ in range(n)))
    prefix = bytes(rng.randrange(256) for _ in range(19))
    for n in range(0, 30):
        for _ in range(3):
            out.append(prefix[:rng.randrange(len(prefix) + 1)] + bytes(rng.choice(alpha) for _ in range(n)))
    return out


def test_string_words_order_as_bytes(host):
    rng = random.Random(7)
    strs = _strings(rng)
    for _ in range(20000):
        a, b = rng.choice(strs), rng.choice(strs)
        assert (_seq(host, a) < _seq(host, b)) == (a < b), (a, b)
        assert (_seq(host, a) == _seq(host, b)) == (a == b), (a, b)
    assert sorted(strs, key=lambda s: _seq(host, s)) == sorted(strs)


def test_padding_and_prefixes(host):
    keys = [b"a", b"a\0", b"a\0\0", b"ab", b"", b"\0", b"a" * 8, b"a" * 8 + b"\0", b"a" * 9, b"a" * 7 + b"\0"]
    assert sorted(keys, key=lambda s: _seq(host, s)) == sorted(keys)
    assert host.h_sort_str_class(0, 0) == 0 and host.h_sort_str_class(8, 0) == 8 and host.h_sort_str_class(9, 0) == 9
    assert host.h_sort_str_class(16, 1) == 8 and host.h_sort_str_class(16, 2) == 0
    assert host.h_sort_str_word(b"\x01\x02", 2, 0) == 0x0102 << 48


@pytest.mark.parametrize("plen", [0, 7, 8, 9, 15, 16, 17, 64, 1000])
def test_lcp_skip_keeps_the_order(host, plen):
    """A tied group of strings that share a prefix jumps by the words every member shares with its first member; comparing from
    there gives the bytes order of the group."""
    rng = random.Random(plen)
    prefix = bytes(rng.randrange(256) for _ in range(plen))
    group = [prefix + bytes(rng.randrange(256) for _ in range(rng.randrange(0, 20))) for _ in range(60)]
    group += [prefix, prefix + b"\0", prefix + b"\xff"]
    first = group[0]
    skip = min(_shared_words(host, g, first, 0) for g in group)
    assert skip >= max(0, plen - 8) // 8  # the shared prefix costs no round
    assert sorted(group, key=lambda s: _seq(host, s, skip)) == sorted(group)


def test_utf8_bytes_order_is_str_order(host):
    rng = random.Random(3)
    chars = ["a", "z", "\x00", "\x7f", "é", "ÿ", "Ā", "€", "￿", "𝄞", "\U0010ffff", "中"]
    strs = ["".join(rng.choice(chars) for _ in range(rng.randrange(0, 12))) for _ in range(3000)]
    by_key = sorted(strs, key=lambda s: _seq(host, s.encode()))
    assert by_key == sorted(strs)


def test_i64_order(host):
    edges = [-(1 << 63), -(1 << 63) + 1, -(1 << 32) - 1, -(1 << 32), -1, 0, 1, (1 << 32) - 1, 1 << 32, (1 << 32) + 1, (1 << 63) - 1]
    rng = random.Random(5)
    vals = edges + [rng.randrange(-(1 << 63), 1 << 63) for _ in range(2000)]
    assert sorted(vals, key=host.h_sort_key_i64) == sorted(vals)
    assert host.h_sort_key_i64(-(1 << 63)) == 0 and host.h_sort_key_i64((1 << 63) - 1) == (1 << 64) - 1
