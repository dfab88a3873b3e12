"""The device id dictionary (surge_b200/csrc/id_dict.cuh) on the CPU, with ids built to share one 64-bit tag (oracle/id_hash.py).

tests/fuzz/id_dict_main.cpp builds the header for the host under ASan + UBSan and runs intern, insert_at and find single-threaded.
Random ids never share a tag, so every probe of the GPU suites stops at its first tag match; here whole clusters share one tag
(3000 ids in one chain, a chain that wraps from the last slot to slot 0, the two ids that hash to 0 and 1 and so both carry tag
1), and each answer must equal a Python dict's. A dictionary filled inside a cluster must keep the rules sgr.h states for a
refused poll: at most max_keys ids, every dense index below that count holds an id that arrived, an admitted id is never
refused, and an id not admitted is refused again.
"""
import os
import struct
import subprocess

import numpy as np
import pytest

from oracle import id_hash as H

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "oracle", "_build")
BIN = os.path.join(OUT, "id_dict_asan")
SRC = os.path.join(ROOT, "tests", "fuzz", "id_dict_main.cpp")
HDR = os.path.join(ROOT, "surge_b200", "csrc", "id_dict.cuh")
DEAD = 0xFFFFFFFF


def _cuda_include():
    from surge_b200 import build as B
    return os.path.join(os.path.dirname(os.path.dirname(os.path.realpath(B._nvcc()))), "include")


@pytest.fixture(scope="module")
def harness():
    os.makedirs(OUT, exist_ok=True)
    if not (os.path.exists(BIN) and os.path.getmtime(BIN) >= max(os.path.getmtime(SRC), os.path.getmtime(HDR))):
        cmd = ["g++", "-std=c++17", "-O1", "-g", "-Wall", "-Wextra", "-fsanitize=address,undefined", "-fno-sanitize-recover=undefined",
               "-fno-omit-frame-pointer", "-I" + _cuda_include(), SRC, "-o", BIN]
        r = subprocess.run(cmd, capture_output=True, text=True)
        if r.returncode != 0:
            if "sanitize" in r.stderr or "asan" in r.stderr.lower():
                pytest.skip("sanitizer build unavailable: " + r.stderr[-300:])
            raise AssertionError(r.stderr[-3000:])
    return BIN


def _ids(ids):
    return struct.pack("<I", len(ids)) + b"".join(struct.pack("<I", len(b)) + b for b in ids)


def _run(tmp_path, mode, body):
    src, dst = tmp_path / f"{mode}.in", tmp_path / f"{mode}.out"
    src.write_bytes(body)
    r = subprocess.run([BIN, mode, str(src), str(dst)], capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-3000:]
    return dst.read_bytes()


def _hashes(tmp_path, ids):
    return np.frombuffer(_run(tmp_path, "hash", _ids(ids)), dtype="<u8").tolist()


def _intern(tmp_path, ops, slots, max_keys, arena_cap):
    """ops: (kind, id) pairs. Returns (answers, ctl0, ctl1, ctl5, ids by dense index below min(ctl0, max_keys))."""
    body = struct.pack("<QQQI", slots, max_keys, arena_cap, len(ops)) + b"".join(struct.pack("<II", k, len(b)) + b for k, b in ops)
    out = _run(tmp_path, "intern", body)
    ans = list(struct.unpack_from(f"<{len(ops)}I", out))
    p = 4 * len(ops)
    c0, c1, c5 = struct.unpack_from("<QQQ", out, p)
    p += 24
    keys = []
    for _ in range(min(c0, max_keys)):
        (n,) = struct.unpack_from("<I", out, p)
        p += 4
        if n == DEAD:
            keys.append(None)
            continue
        keys.append(out[p:p + n])
        p += n
    assert p == len(out)
    return ans, c0, c1, c5, keys


def _index(tmp_path, ids, queries, slots):
    out = _run(tmp_path, "index", struct.pack("<Q", slots) + _ids(ids) + _ids(queries))
    dups, full = struct.unpack_from("<QQ", out)
    return dups, full, np.frombuffer(out[16:], dtype="<i8").tolist()


def _model(ops, max_keys, arena_cap):
    """The dictionary's rules restated: a new id takes its padded bytes, then an index only if the bytes fit; a refused claim
    consumes what it took; a kind-1 op (a refused claim left by a lost race) changes nothing but the slot it kills."""
    known, used, nk, ans = {}, 0, 0, []
    for kind, b in ops:
        if kind == 1:
            ans.append(None)
            continue
        if b in known:
            ans.append(known[b])
            continue
        need = (len(b) + 7) & ~7
        off, used = used, used + need
        if off + need > arena_cap:
            ans.append(DEAD)
            continue
        idx, nk = nk, nk + 1
        if idx >= max_keys:
            ans.append(DEAD)
            continue
        known[b] = idx
        ans.append(idx)
    return ans, nk, used, known


def test_hash_matches_the_restatement(harness, tmp_path):
    rng = np.random.default_rng(1)
    rand = [rng.integers(0, 256, size=n, dtype=np.uint8).tobytes() for n in range(41) for _ in range(25)]
    built = (H.cluster(64, b"c-", seed=2) + H.cluster(16, b"w-", home_mask=(1 << 20) - 1, seed=3) + H.tag_one_pair(b"t-", seed=4)
             + H.cluster(8, b"\x00\xff", length=32, seed=5, alphabet=H.ANY_BYTE) + H.random_ids(200, seed=6))
    built.append(H.near_miss(built[0], seed=7))
    ids = rand + built
    assert _hashes(tmp_path, ids) == [H.hash_id(b) for b in ids]
    # pinned values: the restatement itself must not drift
    assert [H.hash_id(b) for b in (b"", b"a", b"agg-1", b"0123456789abcdef", b"account-000000000042")] == \
        _hashes(tmp_path, [b"", b"a", b"agg-1", b"0123456789abcdef", b"account-000000000042"])
    assert [hex(H.hash_bytes(b)) for b in (b"", b"agg-1")] == [hex(0x90F8749B0FB13233), hex(0x35898D22E4265E57)]


def test_constructed_ids_collide_as_promised():
    c = H.cluster(50, b"c-", seed=11)
    assert len(set(c)) == 50 and len({len(b) for b in c}) == 1 and len({H.hash_id(b) for b in c}) == 1
    assert all(b.startswith(b"c-") and b":" not in b and all(0x20 <= x < 0x7F for x in b) for b in c)
    w = H.cluster(10, b"w-", home_mask=(1 << 20) - 1, seed=12)
    assert H.hash_id(w[0]) & 0xFFFFF == 0xFFFFF
    z, o = H.tag_one_pair(seed=13)
    assert (H.hash_bytes(z), H.hash_bytes(o), H.hash_id(z), H.hash_id(o)) == (0, 1, 1, 1)
    m = H.near_miss(c[0], seed=14)
    hm, hc = H.hash_bytes(m), H.hash_bytes(c[0])
    assert m != c[0] and hm != hc and hm & 0xFFFFFFFF == hc & 0xFFFFFFFF and hm >> 58 == hc >> 58
    for h in (0, 1, 0xFFFFFFFFFFFFFFFF, 0x8000000000000001):
        assert H.unxorshift(h ^ (h >> 29), 29) == h and H.unxorshift(h ^ (h >> 32), 32) == h


def test_intern_over_clusters_is_a_dict(harness, tmp_path):
    rng = np.random.default_rng(21)
    big = H.cluster(3000, b"big-", seed=22)
    wrap = H.cluster(64, b"wrap-", home_mask=(1 << 20) - 1, seed=23)
    pair = H.tag_one_pair(b"one-", seed=24)
    rand = H.random_ids(500, seed=25)
    present = big[:2000] + wrap[:48] + pair[:1] + rand
    seq = [present[i] for i in rng.integers(0, len(present), size=12000)] + present
    rng.shuffle(seq)
    absent = big[2000:] + wrap[48:] + pair[1:] + [H.near_miss(big[0], seed=26)]
    ops = [(0, b) for b in seq] + [(0, b) for b in present]
    for slots in (1024 * 8, 1 << 20):   # wrap's home is the last slot of both tables
        ans, c0, c1, c5, keys = _intern(tmp_path, ops, slots, max_keys=len(present), arena_cap=1 << 20)
        want, nk, used, known = _model(ops, len(present), 1 << 20)
        assert ans == want and (c0, c1, c5) == (nk, used, 0) == (len(present), used, 0)
        assert keys == sorted(known, key=known.get)
        # lookups of ids never interned: each is new, so the next index; read back against the model
        ans2, *_ = _intern(tmp_path, ops + [(0, b) for b in absent], slots, max_keys=len(present) + len(absent), arena_cap=1 << 20)
        assert ans2[len(ops):] == list(range(len(present), len(present) + len(absent)))


def test_insert_at_and_find_over_clusters(harness, tmp_path):
    big = H.cluster(3000, b"idx-", seed=31)
    wrap = H.cluster(100, b"wr-", home_mask=(1 << 20) - 1, seed=32)
    pair = H.tag_one_pair(b"pr-", seed=33)
    rand = H.random_ids(300, seed=34)
    ids = big[:2500] + wrap[:80] + pair[:1] + rand
    rng = np.random.default_rng(35)
    dup_at = sorted(rng.choice(len(ids), size=40, replace=False).tolist())
    with_dups = ids + [ids[i] for i in dup_at]            # true duplicates come after their first copy
    first = {}
    for i, b in enumerate(with_dups):
        first.setdefault(b, i)
    queries = with_dups + big[2500:] + wrap[80:] + pair[1:] + [H.near_miss(big[1], seed=36), b""]
    for slots in (8192, 1 << 14):
        dups, full, got = _index(tmp_path, with_dups, queries, slots)
        assert (dups, full) == (40, 0)
        assert got == [first.get(b, -1) for b in queries]


def test_a_full_dictionary_inside_a_cluster_keeps_its_rules(harness, tmp_path):
    """max_keys and arena bounds reached inside one cluster, with a refused claim's dead slot ahead of admitted members."""
    cl = H.cluster(80, b"full-", seed=41)          # 24-byte ids: 24 arena bytes each
    rand = H.random_ids(10, lengths=(16, 16), seed=42)
    for max_keys, arena_cap in ((40, 1 << 20), (1000, 40 * 24 + 7)):
        ops = [(0, b) for b in rand + cl[:20]]                     # 1: a good poll
        ops += [(1, cl[20])]                                       # a claim that lost the race for the last index, ahead of ...
        ops += [(0, b) for b in cl[21:60]]                         # 2: ... members admitted behind it, then the bound
        ops += [(0, b) for b in rand + cl[:60]]                    # 3: everything seen so far, again
        ops += [(0, cl[20]), (0, cl[70])]                          # 4: a refused and a never-seen id
        ans, c0, c1, c5, keys = _intern(tmp_path, ops, 1024, max_keys, arena_cap)
        want, nk, used, known = _model(ops, max_keys, arena_cap)
        assert [a for a, (k, _) in zip(ans, ops) if k == 0] == [w for w, (k, _) in zip(want, ops) if k == 0]
        admitted = sorted(known, key=known.get)
        assert 0 < len(admitted) < 60 and len(admitted) <= max_keys
        assert sum(len(b) for b in admitted) <= arena_cap
        assert keys[:len(admitted)] == admitted                   # every index below the clamped count holds an arrived id
        assert len(keys) == min(c0, max_keys) == len(admitted)
        refused = {b for (k, b), a in zip(ops, ans) if k == 0 and a == DEAD}
        assert refused and not refused & set(admitted) and cl[20] in refused and cl[70] in refused
        assert c5 == 1 + sum(1 for (k, _), a in zip(ops, ans) if k == 0 and a == DEAD)
        # every admitted id, including those behind the dead slot, reads back at its index
        again = [a for (k, b), a in zip(ops, ans) if k == 0 and b in known]
        assert again == [known[b] for k, b in ops if k == 0 and b in known]
