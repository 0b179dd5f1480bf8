"""numpy uint64 restatements of the hashes behind the library's open-addressed tables, their inverses, the table-size
rules, and generators of keys that collide in those tables.

Every table probes linearly from a home slot taken from its hash, so keys with one hash (or one home slot) form one
probe chain.  The generators build such chains on purpose: most of the hashes are bijections one can run backwards.

- key_hash (kernels.cuh:1280): xor / odd multiply / xorshift per 64-bit word, then a final mix.  Choose the first
  three words of a 32-byte key and solve for the last one: any target hash.
- join_hash (kernels.cuh:995): the splitmix64 finaliser over `chat * C ^ msg`.  Invert the finaliser, pick any chat and
  `msg = x ^ chat * C` (or any msg and solve for chat).
- st_hash (state.cuh:65): join_hash with the (row, gen) mix xored into chat, so keys differing in row or generation
  can share one full hash.
- la_hash (local_appends.cuh:59) and usernames (only [a-z0-9]) need only the low bits of a slot: brute force.

tests/hash_check.cu evaluates the device functions on the generators' inputs; test_gpu_hash_collisions.py drives the
tables with them."""
from __future__ import annotations

import numpy as np

M64 = (1 << 64) - 1
PHI = 0x9E3779B97F4A7C15
KH_M, KH_F = 0xFF51AFD7ED558CCD, 0xC4CEB9FE1A85EC53
SM_1, SM_2 = 0xBF58476D1CE4E5B9, 0x94D049BB133111EB
ST_MIX = 0x632BE59BD9B4E019
FNV_OFF, FNV_PRIME = 0xCBF29CE484222325, 0x100000001B3
INT64_MIN, INT64_MAX = -(1 << 63), (1 << 63) - 1
U = np.uint64


def _u(x):
    return np.asarray(x).astype(np.uint64)


def _i64(x: int) -> int:
    x &= M64
    return x - (1 << 64) if x >> 63 else x


# ---- table sizes: every rule as the library's host code computes it --------------------------------------------------
def next_pow2(v: int) -> int:  # tgingest.cu:516
    p = 1
    while p < v:
        p <<= 1
    return p


def set_table_slots(cap: int) -> int:
    """a key set of `cap` keys (tgingest.cu:2134 the dedup set, :676 a growth step, :2530 an exclusion set's first add);
    also set_info()["table_slots"]"""
    return next_pow2(2 * cap)


def grown_capacity(count: int, need: int, grow_max: int) -> int:  # tgingest.cu:676
    return min(next_pow2(count + need), grow_max)


def frontier_batch_slots(links: int) -> int:  # tgingest.cu:588
    return next_pow2(max(2 * links, 1024))


def join_slots(na: int) -> int:  # tgingest.cu:2309
    return next_pow2(max(2 * na, 1024))


STATE_INITIAL_SLOTS = 1024  # tgingest.cu:3506


def state_table_slots(tslots: int, need: int) -> int:
    """the message table after room for `need` message rows is reserved (tgingest.cu:3615)"""
    return next_pow2(max(4 * need, 1024)) if 2 * need > tslots else tslots


def state_batch_slots(m: int) -> int:  # tgingest.cu:3927 (UpdateMessage), :4727 (turn), :4962 (view)
    return next_pow2(max(2 * m, 64))


def sink_slots(rows: int) -> int:  # tgingest.cu:2739
    return next_pow2(max(2 * rows, 64))


# ---- key_hash and the slots it feeds --------------------------------------------------------------------------------
def key_words(keys: np.ndarray) -> np.ndarray:
    """(n, 32) uint8 -> (n, 4) uint64: word i = bytes 8i..8i+7, little endian (Key32 w[2i] | w[2i+1] << 32)"""
    return np.ascontiguousarray(keys, np.uint8).reshape(-1, 32).view("<u8")


@np.errstate(over="ignore")
def key_hash(keys: np.ndarray) -> np.ndarray:  # kernels.cuh:1280
    x = key_words(keys)
    h = np.full(len(x), PHI, U)
    for i in range(4):
        h = (h ^ x[:, i]) * U(KH_M)
        h ^= h >> U(32)
    h = h * U(KH_F)
    return h ^ (h >> U(29))


def set_fp(h):  # kernels.cuh:1295: 24-bit fingerprint, never 0
    return (_u(h) >> U(40)) | U(1)


def set_home(h, tslots: int):  # kernels.cuh:1296
    return _u(h) & U(tslots - 1)


def batch_slot(h, bslots: int):  # kernels.cuh:1369 (frontier batch), state.cuh st_first_kernel (candidates)
    return (_u(h) >> U(7)) & U(bslots - 1)


def key_owner(h, nranks: int):  # kernels.cuh:1471
    return ((_u(h) >> U(17)) % U(nranks)).astype(np.uint32)


@np.errstate(over="ignore")
def st_first_hash(h, span, per_span: bool):  # state.cuh st_cand_hash
    return _u(h) ^ (_u(span) * U(PHI) if per_span else U(0))


# ---- join_hash, st_hash and their slots -----------------------------------------------------------------------------
@np.errstate(over="ignore")  # uint64 arithmetic wraps, as on the device; numpy scalars would warn
def _fin(x):
    x = x ^ (x >> U(30))
    x = x * U(SM_1)
    x = x ^ (x >> U(27))
    x = x * U(SM_2)
    return x ^ (x >> U(31))


@np.errstate(over="ignore")
def join_hash(chat, msg):  # kernels.cuh:995
    return _fin(np.asarray(chat, np.int64).view(U) * U(PHI) ^ np.asarray(msg, np.int64).view(U))


@np.errstate(over="ignore")
def st_mix(row, gen):
    return ((_u(row) << U(32)) | _u(gen)) * U(ST_MIX)


def st_hash(row, gen, chat, msg):  # state.cuh:65
    return join_hash((np.asarray(chat, np.int64).view(U) ^ st_mix(row, gen)).view(np.int64), msg)


def st_turn_slot(k, msg, bslots: int):  # state.cuh:197
    return st_hash(k, 0, np.zeros_like(np.asarray(msg, np.int64)), msg) & U(bslots - 1)


def st_view_slot(pg, chat, msg, vslots: int):  # state.cuh:320
    return st_hash(pg, 0, chat, msg) & U(vslots - 1)


# ---- la_hash (the local sink's channelID table) ----------------------------------------------------------------------
def la_hash(name: bytes) -> int:  # local_appends.cuh:59
    h = FNV_OFF ^ len(name)
    for b in name:
        h = ((h ^ b) * FNV_PRIME) & M64
    return h ^ (h >> 31)


@np.errstate(over="ignore")
def la_hash_many(names: np.ndarray, length: int) -> np.ndarray:
    """la_hash of n names of one length, given as (n, length) uint8"""
    h = np.full(len(names), FNV_OFF ^ length, U)
    for k in range(length):
        h = (h ^ names[:, k].astype(U)) * U(FNV_PRIME)
    return h ^ (h >> U(31))


# ---- inverses (Python ints) ------------------------------------------------------------------------------------------
def inv_mul(m: int) -> int:
    return pow(m, -1, 1 << 64)


def unxorshift(y: int, s: int) -> int:
    """the x with x ^ (x >> s) == y"""
    x = y
    for _ in range(64 // s + 1):
        x = y ^ (x >> s)
    return x & M64


def fin_inv(h: int) -> int:
    """the x with _fin(x) == h"""
    x = unxorshift(h, 31)
    x = (x * inv_mul(SM_2)) & M64
    x = unxorshift(x, 27)
    x = (x * inv_mul(SM_1)) & M64
    return unxorshift(x, 30)


def key_hash_state(words3) -> int:
    """the running hash after the first three words"""
    h = PHI
    for x in words3:
        h = ((h ^ int(x)) * KH_M) & M64
        h ^= h >> 32
    return h


def key_last_word(words3, target: int) -> int:
    """the fourth word that makes key_hash equal target, given the first three"""
    y = unxorshift(target, 29)
    y = (y * inv_mul(KH_F)) & M64
    y = unxorshift(y, 32)
    y = (y * inv_mul(KH_M)) & M64
    return y ^ key_hash_state(words3)


def join_msg_for(chat: int, target: int) -> int:
    """the msg with join_hash(chat, msg) == target"""
    return _i64(fin_inv(target) ^ ((chat & M64) * PHI))


def join_chat_for(msg: int, target: int) -> int:
    """the chat with join_hash(chat, msg) == target"""
    return _i64(((fin_inv(target) ^ (msg & M64)) * inv_mul(PHI)))


def st_msg_for(row: int, gen: int, chat: int, target: int) -> int:
    """the msg with st_hash(row, gen, chat, msg) == target"""
    c = (chat & M64) ^ ((((row << 32) | gen) * ST_MIX) & M64)
    return join_msg_for(_i64(c), target)


# ---- generators --------------------------------------------------------------------------------------------------
def keys_with_hash(n: int, target: int, prefix: bytes = b"", vary_first: bool = False) -> np.ndarray:
    """n distinct 32-byte keys whose key_hash is target: bytes [0, 24) chosen (prefix, then a counter), bytes [24, 32)
    solved.  vary_first: the keys differ only in byte 0 before the solved word (n <= 255), byte 0 never 0"""
    assert len(prefix) <= 20
    keys = np.zeros((n, 32), np.uint8)
    if vary_first:
        assert n <= 255
        keys[:, 1:24] = np.frombuffer(b"k" * 23, np.uint8)
        keys[:, 0] = np.arange(1, n + 1)
    else:
        keys[:, :len(prefix)] = np.frombuffer(prefix, np.uint8)
        c = np.arange(n, dtype=np.uint32)
        keys[:, 20:24] = c.view(np.uint8).reshape(n, 4)
        keys[:, len(prefix):20] = ord("x")
    w = key_words(keys)
    for i in range(n):
        w[i, 3] = key_last_word(w[i, :3], target)
    return keys


def keys_last_byte(tslots: int, first: int, span: int, rng) -> np.ndarray:
    """>= 2 keys that differ only in byte 31, each with its home slot in the span of `span` slots from `first` (mod
    tslots), where a crafted chain lies.  Keys that differ in one byte never share a full hash (each word enters
    key_hash through a bijection), nor, in practice, a home slot: they differ in fingerprint, and a probe for one must
    walk past the chain and the others."""
    inside = (np.arange(tslots) - first) % tslots < span
    while True:
        k = np.repeat(rng.integers(1, 256, (1, 32), dtype=np.uint8), 256, 0)
        k[:, 31] = np.arange(256, dtype=np.uint8)
        hit = k[inside[set_home(key_hash(k), tslots).astype(np.int64)]]
        if len(hit) >= 2:
            return hit


def _mask_bits(tslots: int, bslots: int) -> int:
    return (tslots - 1) | ((bslots - 1) << 7)


USER_HEAD = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz", np.uint8)
USER_TAIL = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789", np.uint8)


def usernames_colliding(n: int, tslots: int, bslots: int, target: int, rng, length: int = 12) -> list[bytes]:
    """n distinct usernames (a letter, then [a-z0-9]: valid 5-32 byte Telegram usernames) whose zero-padded 32-byte
    keys share target's home slot in a set of tslots slots and its batch slot in a frontier batch table of bslots"""
    assert 5 <= length <= 32
    mask = U(_mask_bits(tslots, bslots))
    want = U(target) & mask
    out: dict[bytes, None] = {}
    while len(out) < n:
        m = 1 << 20
        k = np.zeros((m, 32), np.uint8)
        k[:, 0] = rng.choice(USER_HEAD, m)
        k[:, 1:length] = rng.choice(USER_TAIL, (m, length - 1))
        hit = k[(key_hash(k) & mask) == want]
        for row in hit:
            out.setdefault(row[:length].tobytes())
    return list(out)[:n]


def join_pairs(n: int, target: int, rng, ends: bool = True) -> np.ndarray:
    """n distinct (chat, msg) int64 pairs with join_hash == target; with ends, chats and msgs at the int64 ends first"""
    out: dict[tuple, None] = {}
    if ends:
        for v in (INT64_MIN, INT64_MAX, INT64_MIN + 1, INT64_MAX - 1, -1, 0, 1):
            out.setdefault((v, join_msg_for(v, target)))
            out.setdefault((join_chat_for(v, target), v))
    while len(out) < n:
        c = _i64(int(rng.integers(0, 1 << 63)) * 2 + int(rng.integers(0, 2)))
        out.setdefault((c, join_msg_for(c, target)))
    return np.array(list(out)[:n], np.int64).reshape(-1, 2)


def st_tuples(n: int, target: int, rows, gens, rng) -> list[tuple[int, int, int, int]]:
    """n distinct (row, gen, chat, msg) with st_hash == target, cycling over rows and gens"""
    out: dict[tuple, None] = {}
    k = 0
    while len(out) < n:
        row, gen = rows[k % len(rows)], gens[(k // len(rows)) % len(gens)]
        chat = -1001000000000 - int(rng.integers(0, 1 << 30))
        out.setdefault((row, gen, chat, st_msg_for(row, gen, chat, target)))
        k += 1
    return list(out)[:n]


def st_same_home_across_gens(n: int, row: int, gens, chat: int, bits: int, rng, slot: int | None = None) -> list[int]:
    """n distinct msgs whose (row, g, chat, msg) keys share one home slot in every table of <= 2^bits slots for every g
    in gens (and, if slot is given, home slot `slot` there)"""
    mask = U((1 << bits) - 1)
    out: list[int] = []
    while len(out) < n:
        m = rng.integers(1, 1 << 40, 1 << 20, dtype=np.int64)
        hs = [st_hash(np.full(len(m), row, U), np.full(len(m), g, U), np.full(len(m), chat, np.int64), m) & mask
              for g in gens]
        ok = np.ones(len(m), bool)
        for h in hs[1:]:
            ok &= h == hs[0]
        if slot is not None:
            ok &= hs[0] == U(slot)
        out += [int(v) for v in m[ok] if int(v) not in out]
    return out[:n]


def st_batch_collisions(n: int, bslots: int, slot: int, rows, chat: int, rng) -> list[tuple[int, int]]:
    """n distinct (row, msg) whose UpdateMessage keys (row, chat, msg) share batch slot `slot` of a table of bslots"""
    out: dict[tuple, None] = {}
    mask = U(bslots - 1)
    while len(out) < n:
        m = rng.integers(1, 1 << 40, 1 << 18, dtype=np.int64)
        r = np.asarray(rows, np.uint64)[rng.integers(0, len(rows), len(m))]
        ok = (st_hash(r, np.zeros(len(m), U), np.full(len(m), chat, np.int64), m) & mask) == U(slot)
        for rr, mm in zip(r[ok], m[ok]):
            out.setdefault((int(rr), int(mm)))
    return list(out)[:n]


def la_names_colliding(n: int, tslots: int, slot: int, rng, lengths=(1, 3, 8, 20)) -> list[bytes]:
    """n distinct channel names of the given lengths ([a-z0-9_] bytes) with la_hash home slot `slot` in tslots slots"""
    out: dict[bytes, None] = {}
    mask = U(tslots - 1)
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789_", np.uint8)
    k = 0
    while len(out) < n:
        L = lengths[k % len(lengths)]
        k += 1
        c = rng.choice(alpha, (1 << 16, L))
        for row in c[(la_hash_many(c, L) & mask) == U(slot)][:4]:
            out.setdefault(row.tobytes())
    return list(out)[:n]


def la_prefix_chain(depth: int, tslots: int, slot: int, rng, start: bytes = b"") -> list[bytes]:
    """names n_0, n_1, ... each a proper prefix of the next, all with home slot `slot` in tslots slots; n_0 may be the
    empty name when `start` is b"" and it lands there"""
    alpha = np.frombuffer(b"abcdefghijklmnopqrstuvwxyz0123456789_", np.uint8)
    mask = U(tslots - 1)
    out = [start] if (la_hash(start) & (tslots - 1)) == slot else []
    cur = start
    while len(out) < depth:
        tail = rng.choice(alpha, (1 << 14, 3))
        c = np.concatenate([np.repeat(np.frombuffer(cur, np.uint8).reshape(1, -1), len(tail), 0), tail], 1)
        hit = c[(la_hash_many(c, c.shape[1]) & mask) == U(slot)]
        cur = hit[0].tobytes()
        out.append(cur)
    return out


def wrap_target(bits: int = 30, high: int = 0x5EED) -> int:
    """a hash whose low `bits` bits are all ones: home slot tmask in every table of <= 2^bits slots, and batch slot
    bmask in every batch table of <= 2^(bits - 7) slots, so the chain wraps to slot 0"""
    return ((high << bits) | ((1 << bits) - 1)) & M64
