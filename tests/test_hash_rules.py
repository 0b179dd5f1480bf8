"""The hash restatements of tests/hash_rules.py on the CPU: every inverse runs its hash backwards, and every generator's
keys really collide under the restatement at the table sizes they are made for.  tests/hash_check.cu compares the
restatements with the device functions."""
import numpy as np
import pytest

import hash_rules as hr


def test_inverses_round_trip():
    rng = np.random.default_rng(1)
    for v in [0, 1, hr.M64, hr.PHI] + [int(x) for x in rng.integers(0, 1 << 63, 200, dtype=np.int64)]:
        for s in (27, 29, 30, 31, 32):
            assert hr.unxorshift(v ^ (v >> s), s) == v
        assert hr.fin_inv(int(hr._fin(np.array([v], np.uint64))[0])) == v
        x = hr.fin_inv(v)
        assert int(hr._fin(np.array([x], np.uint64))[0]) == v
    for m in (hr.KH_M, hr.KH_F, hr.SM_1, hr.SM_2, hr.PHI):
        assert (m * hr.inv_mul(m)) & hr.M64 == 1


def test_key_last_word_gives_any_hash():
    rng = np.random.default_rng(2)
    keys = rng.integers(0, 256, (64, 32), dtype=np.uint8)
    targets = [int(t) for t in rng.integers(0, 1 << 63, 64, dtype=np.int64)]
    w = hr.key_words(keys)
    for i, t in enumerate(targets):
        w[i, 3] = hr.key_last_word(w[i, :3], t)
    assert [int(h) for h in hr.key_hash(keys)] == targets


@pytest.mark.parametrize("n", [2, 33, 1000, 4096])
def test_keys_with_hash_collide(n):
    t = hr.wrap_target()
    for prefix in (b"", b"channel_"):
        k = hr.keys_with_hash(n, t, prefix)
        assert len({r.tobytes() for r in k}) == n
        assert (k[:, :len(prefix)] == np.frombuffer(prefix, np.uint8)).all()
        assert (hr.key_hash(k) == np.uint64(t)).all()
    k = hr.keys_with_hash(min(n, 255), t, vary_first=True)
    assert (k[:, 1:24] == k[0, 1:24]).all() and len(set(k[:, 0])) == len(k)
    assert (hr.key_hash(k) == np.uint64(t)).all()


def test_keys_differing_in_the_last_byte_land_in_a_chain():
    g = hr.keys_last_byte(2048, 2047, 34, np.random.default_rng(8))
    assert len(g) >= 2 and (g[:, :31] == g[0, :31]).all() and len(set(g[:, 31])) == len(g)
    home = hr.set_home(hr.key_hash(g), 2048).astype(np.int64)
    assert ((home - 2047) % 2048 < 34).all()


def test_wrap_target_wraps_every_table():
    t = hr.wrap_target()
    for slots in (64, 1024, 1 << 16, 1 << 23):
        assert int(hr.set_home(t, slots)) == slots - 1
        assert int(hr.batch_slot(t, slots)) == slots - 1


def test_usernames_collide_in_the_set_and_the_batch_table():
    rng = np.random.default_rng(3)
    t = hr.wrap_target()
    names = hr.usernames_colliding(40, 1 << 13, 1024, t, rng)
    assert len(set(names)) == 40
    for nm in names:
        assert 5 <= len(nm) <= 32 and nm[:1].isalpha() and all(c in b"abcdefghijklmnopqrstuvwxyz0123456789" for c in nm)
    from distributed_crawler_b200.engine import names_to_keys32
    h = hr.key_hash(names_to_keys32(names))
    assert (hr.set_home(h, 1 << 13) == np.uint64((1 << 13) - 1)).all()
    assert (hr.batch_slot(h, 1024) == np.uint64(1023)).all()
    assert (hr.set_home(h, 1 << 12) == np.uint64((1 << 12) - 1)).all()  # and every smaller table


def test_join_pairs_collide_with_the_int64_ends():
    rng = np.random.default_rng(4)
    t = hr.wrap_target()
    p = hr.join_pairs(300, t, rng)
    assert len({tuple(r) for r in p}) == 300
    assert (hr.join_hash(p[:, 0], p[:, 1]) == np.uint64(t)).all()
    for v in (hr.INT64_MIN, hr.INT64_MAX):
        assert (p[:, 0] == v).any() and (p[:, 1] == v).any()
    c, m = 0x123456789, hr.join_msg_for(0x123456789, 77)
    assert int(hr.join_hash(c, m)) == 77 and int(hr.join_hash(hr.join_chat_for(m, 99), m)) == 99


def test_st_tuples_collide_across_rows_and_generations():
    rng = np.random.default_rng(5)
    t = hr.wrap_target()
    q = hr.st_tuples(100, t, rows=[0, 1, 7, 1 << 20], gens=[0, 1, 2], rng=rng)
    a = np.array(q, dtype=object)
    h = hr.st_hash(a[:, 0].astype(np.uint64), a[:, 1].astype(np.uint64), a[:, 2].astype(np.int64), a[:, 3].astype(np.int64))
    assert (h == np.uint64(t)).all()
    assert len({r for r, *_ in q}) == 4 and len({g for _, g, *_ in q}) == 3
    # one (chat, msg) under several generations of one row: one home slot in every table of <= 2^14 slots
    ms = hr.st_same_home_across_gens(6, 3, (0, 1), -100, 12, rng)
    for bits in (10, 12):
        for m in ms:
            assert len({int(hr.st_hash(3, g, -100, m)) & ((1 << bits) - 1) for g in (0, 1)}) == 1
    ms = hr.st_same_home_across_gens(2, 3, (0, 1), -100, 10, rng, slot=1023)
    assert all(int(hr.st_hash(3, g, -100, m)) & 1023 == 1023 for g in (0, 1) for m in ms)


def test_st_batch_turn_and_view_slots():
    rng = np.random.default_rng(6)
    rm = hr.st_batch_collisions(50, 128, 127, rows=[0, 1, 2], chat=-5, rng=rng)
    assert len(set(rm)) == 50
    for row, m in rm:
        assert int(hr.st_hash(row, 0, -5, m)) & 127 == 127
    m = np.arange(-3, 300, dtype=np.int64)
    assert (hr.st_turn_slot(np.full(len(m), 4, np.uint64), m, 256) == hr.st_hash(4, 0, 0, m) & np.uint64(255)).all()
    assert (hr.st_view_slot(2, -7, m, 64) == hr.st_hash(2, 0, -7, m) & np.uint64(63)).all()


def test_st_first_per_span_mix():
    k = hr.keys_with_hash(4, hr.wrap_target())
    h = hr.key_hash(k)
    assert (hr.st_first_hash(h, np.arange(4), False) == h).all()
    got = hr.st_first_hash(h, np.arange(4), True)
    assert int(got[0]) == int(h[0]) and len(set(got.tolist())) == 4


def test_la_names_collide():
    rng = np.random.default_rng(7)
    for tslots, slot in ((64, 63), (128, 5), (1024, 1023)):
        names = hr.la_names_colliding(30, tslots, slot, rng)
        assert len(set(names)) == 30
        assert all(hr.la_hash(nm) & (tslots - 1) == slot for nm in names)
        many = np.frombuffer(b"".join(n for n in names if len(n) == 8), np.uint8).reshape(-1, 8)
        assert [int(h) for h in hr.la_hash_many(many, 8)] == [hr.la_hash(n) for n in names if len(n) == 8]
    slot = hr.la_hash(b"") & 127
    chain = hr.la_prefix_chain(5, 128, slot, rng)
    assert chain[0] == b"" and all(chain[i + 1].startswith(chain[i]) and len(chain[i + 1]) > len(chain[i]) for i in range(4))
    assert all(hr.la_hash(nm) & 127 == slot for nm in chain)


def test_table_size_rules():
    assert [hr.next_pow2(v) for v in (0, 1, 2, 3, 1024, 1025)] == [1, 1, 2, 4, 1024, 2048]
    assert hr.set_table_slots(1000) == 2048 and hr.set_table_slots(64) == 128
    assert hr.frontier_batch_slots(10) == 1024 and hr.frontier_batch_slots(600) == 2048
    assert hr.join_slots(0) == 1024 and hr.join_slots(4096) == 8192
    assert hr.state_table_slots(1024, 512) == 1024 and hr.state_table_slots(1024, 513) == 4096
    assert hr.state_batch_slots(3) == 64 and hr.sink_slots(33) == 128
    assert hr.grown_capacity(64, 1, 1 << 20) == 128 and hr.grown_capacity(1000, 5000, 4096) == 4096


def test_key_owner_is_bits_17_up():
    h = np.array([0, 1 << 17, 5 << 17, hr.M64], np.uint64)
    assert hr.key_owner(h, 4).tolist() == [0, 1, 1, ((hr.M64 >> 17) % 4)]
