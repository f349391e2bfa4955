"""Kernel by kernel against plain references: the emitter (ck_emit_kernel), the offset scan (ck_scan_*) and the Kafka key
hash (ck_murmur2_key through the plan's shared-memory window PRd and the route kernel's global reader GRd), run through
the launchers of tests/devsim on inputs made here.  The producers only ever hand these kernels a narrow set of inputs;
these tests cover the contract they document: segments of any length (empty ones included) at any byte, offsets past
2^32, keys of any length and alignment with every escape a canonical record can hold."""
import json
import random

import numpy as np
import pytest

from test_gpu_parity import _murmur2

pytestmark = pytest.mark.gpu

DESC = np.dtype([("nseg", "<u4"), ("record", "<u4"), ("total_len", "<u4"), ("pad", "<u4"), ("seg", "<u4", (16, 2))])
INPUT, LIT, AUX, GLUE = 0, 1, 2, 3
GLUE_STRIDE = 512
SLACK = 32          # bytes after every source buffer (the emitter may read 19 past a segment's end)
MARK = 0xEE         # what the slack holds: a marker that must never reach an output
CANARY = 0xA5       # what the output holds before the launch


@pytest.fixture(scope="module")
def dev():
    import torch
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    import devsim
    return devsim.lib()


def _cuda(a: np.ndarray):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _with_slack(b: np.ndarray) -> np.ndarray:
    return np.concatenate([b.astype(np.uint8), np.full(SLACK, MARK, np.uint8)])


# ---------------------------------------------------------------------------------------------------------------------
# emitter
# ---------------------------------------------------------------------------------------------------------------------
def _seg_len(rng) -> int:
    c = rng.random()
    if c < 0.35:
        return rng.randrange(0, 18)
    if c < 0.5:
        return rng.randrange(31, 34)
    if c < 0.65:
        return rng.randrange(47, 50)
    return rng.randrange(0, 601)


def _random_layout(rng) -> list[tuple[int, int]]:
    return [(rng.randrange(4), _seg_len(rng)) for _ in range(rng.randrange(1, 17))]


def _aligned_layout(rng, empty_at: str | None) -> list[tuple[int, int]]:
    """SegWriter's layout: every segment starts on a 16-byte vector of the payload, all but the last are whole vectors;
    optionally with an empty segment first, in the middle or last"""
    n = rng.randrange(1, 16 if empty_at else 17)
    segs = [(rng.randrange(4), 16 * rng.randrange(1, 33)) for _ in range(n - 1)] + [(rng.randrange(4), rng.randrange(1, 601))]
    if empty_at == "first":
        segs.insert(0, (rng.randrange(4), 0))
    elif empty_at == "middle":
        segs.insert(rng.randrange(1, len(segs)) if len(segs) > 1 else 0, (rng.randrange(4), 0))
    elif empty_at == "last":
        segs.append((rng.randrange(4), 0))
    return segs


def _emit_case(seed: int, n_random: int):
    """sources, descriptors and the expected payloads"""
    rng = random.Random(seed)
    nrec = 97
    rec_len = [rng.randrange(640, 3000) for _ in range(nrec)]
    rec_off = np.zeros(nrec + 1, np.int64)
    rec_off[1:] = np.cumsum(rec_len)
    nprng = np.random.default_rng(seed)
    src = {INPUT: nprng.integers(0, 256, int(rec_off[-1]), dtype=np.uint8),
           LIT: nprng.integers(0, 256, 4001, dtype=np.uint8), AUX: nprng.integers(0, 256, 5003, dtype=np.uint8)}

    layouts = [_random_layout(rng) for _ in range(n_random)]
    layouts += [_aligned_layout(rng, where) for where in (None, "first", "middle", "last") for _ in range(600)]
    layouts += [[(rng.randrange(4), 1) for _ in range(16)] for _ in range(200)]                      # one vector, 16 segments
    layouts += [[(rng.randrange(4), rng.randrange(2, 30))] + [(rng.randrange(4), 1) for _ in range(15)] for _ in range(200)]
    layouts += [[(rng.randrange(4), 32), (rng.randrange(4), 0), (rng.randrange(4), 20)],            # the empty segment
                [(rng.randrange(4), 0), (rng.randrange(4), 20)]] * 50                                # starts a vector
    layouts += [[(INPUT, 0)], [(LIT, 0), (AUX, 0)], []] * 20                                        # empty payloads
    rng.shuffle(layouts)
    layouts += [[(GLUE, 40), (INPUT, 17), (GLUE, 33)]]  # the last glue slot: its segments end on the buffer's last byte
    layouts += [[(AUX, 100), (LIT, 7)]] * 3          # the last three do not fit out_cap below: never written
    n = len(layouts)
    src[GLUE] = nprng.integers(0, 256, (n - 3) * GLUE_STRIDE, dtype=np.uint8)

    descs = np.zeros(n, DESC)
    want = []
    ends_at_buffer_end = set()
    residues = {s: set() for s in range(4)}
    for i, segs in enumerate(layouts):
        rec = nrec - 1 if rng.random() < 0.05 else rng.randrange(nrec)
        parts = []
        for k, (s, ln) in enumerate(segs):
            if s == GLUE:
                ln = min(ln, GLUE_STRIDE)
                lo, hi = i * GLUE_STRIDE, (i + 1) * GLUE_STRIDE
            elif s == INPUT:
                lo, hi = int(rec_off[rec]), int(rec_off[rec + 1])
            else:
                lo, hi = 0, len(src[s])
            at_end = rng.random() < 0.1 or i == n - 4                                 # some end on the source's last byte
            a = hi - ln if at_end else rng.randrange(lo, hi - ln + 1)
            if a + ln == len(src[s]):
                ends_at_buffer_end.add(s)
            residues[s].add(a % 16)
            descs["seg"][i, k] = (a - lo if s in (INPUT, GLUE) else a, (ln << 2) | s)
            parts.append(src[s][a:a + ln])
        payload = np.concatenate(parts) if parts else np.zeros(0, np.uint8)
        descs["nseg"][i], descs["record"][i], descs["total_len"][i] = len(segs), rec, len(payload)
        want.append(payload)
    assert ends_at_buffer_end == {INPUT, LIT, AUX, GLUE} and all(len(r) == 16 for r in residues.values())
    return layouts, rec_off, {s: _with_slack(b) for s, b in src.items()}, descs, want


def _emit(dev, rec_off, src, descs, out_off, out_cap):
    import devsim
    t = {s: _cuda(b) for s, b in src.items()}
    d_off, d_descs, d_out_off = _cuda(rec_off), _cuda(descs.view(np.uint8)), _cuda(out_off)
    out = _cuda(np.full(int(out_off[-1]) + 256, CANARY, np.uint8))
    devsim.check(dev.ck_dev_emit(t[INPUT].data_ptr(), d_off.data_ptr(), len(rec_off) - 1, t[LIT].data_ptr(), t[AUX].data_ptr(),
                                 t[GLUE].data_ptr(), d_descs.data_ptr(), d_out_off.data_ptr(), len(descs), out.data_ptr(), out_cap))
    return out.cpu().numpy()


def test_emit_random_descriptors_match_concatenation(dev):
    """20,000+ payloads of 0-16 segments from all four sources: lengths 0-17, 31-33, 47-49 and up to 600 at every source
    residue, some ending on the last byte of their buffer, payloads over 512 B, a vector of 16 one-byte segments, and the
    aligned layout with empty segments first, in the middle and last.  Bytes [out_off, out_off + total_len) of every
    payload equal the concatenation of its segments; nothing past the last payload that fits out_cap is written."""
    layouts, rec_off, src, descs, want = _emit_case(seed=11, n_random=18000)
    n = len(descs)
    assert n >= 20000 and sum(len(w) > 512 for w in want) > 2000
    lens = np.array([len(w) for w in want], np.int64)
    out_off = np.zeros(n + 1, np.int64)
    out_off[1:] = np.cumsum((lens + 15) & ~15)
    out_cap = int(out_off[n - 3])             # the last three payloads end beyond the capacity
    got = _emit(dev, rec_off, src, descs, out_off, out_cap)
    bad = [i for i in range(n - 3) if not np.array_equal(got[out_off[i]:out_off[i] + lens[i]], want[i])]
    assert not bad, [(i, [(s, ln) for s, ln in layouts[i]]) for i in bad[:12]] + [f"{len(bad)} payloads differ"]
    assert (got[out_cap:] == CANARY).all(), "bytes written past the last payload that fits out_cap"


# ---------------------------------------------------------------------------------------------------------------------
# scan
# ---------------------------------------------------------------------------------------------------------------------
TILE, BLOCK = 2048, 256


@pytest.mark.parametrize("pad", [15, 0])
@pytest.mark.parametrize("n", [1, TILE - 1, TILE, TILE + 1, BLOCK * TILE - 1, BLOCK * TILE, BLOCK * TILE + 1])
def test_scan_offsets_match_int64_cumsum(dev, n, pad):
    """out_off = exclusive int64 prefix sum of the padded lengths, out_off[n] the total, and the grand total, for lengths
    up to 2^31 (totals far past 2^32) at one tile +- 1 and at 256 tiles +- 1 (the tile-sum kernel's loop runs twice)"""
    import torch
    import devsim
    rng = np.random.default_rng(n * 31 + pad)
    lens = rng.integers(0, 1 << 31, n, dtype=np.uint32)
    small = rng.random(n) < 0.3
    lens[small] = rng.integers(0, 40, int(small.sum()), dtype=np.uint32)
    padded = (lens.astype(np.int64) + pad) & ~pad
    want = np.zeros(n + 1, np.int64)
    want[1:] = np.cumsum(padded)
    d_len = _cuda(lens.view(np.int32))
    out = torch.full((n + 2,), -7, dtype=torch.int64, device="cuda")
    tile_sum = torch.zeros(n // TILE + 2, dtype=torch.int64, device="cuda")
    grand = torch.zeros(1, dtype=torch.int64, device="cuda")
    devsim.check(dev.ck_dev_scan(d_len.data_ptr(), n, out.data_ptr(), pad, tile_sum.data_ptr(), grand.data_ptr()))
    got = out.cpu().numpy()
    bad = np.flatnonzero(got[:n + 1] != want)
    assert bad.size == 0, (bad[:8], got[bad[:8]], want[bad[:8]])
    assert got[n + 1] == -7 and int(grand.item()) == want[n]
    if n > TILE:
        assert want[n] > 1 << 32


# ---------------------------------------------------------------------------------------------------------------------
# key hash
# ---------------------------------------------------------------------------------------------------------------------
_SPELL = None


def _spellings() -> dict[str, bytes]:
    """the raw JSON spelling of every character a canonical record escapes, as oracle.port.encode writes it"""
    global _SPELL
    if _SPELL is None:
        from calfkit import synth
        from oracle import port
        obj = json.loads(synth.tool_events(1, seed=1)[0])
        chars = [chr(c) for c in range(0x20)] + ['"', "\\"]
        ids = []
        for c in chars:
            obj["context"]["deps"]["correlation_id"] = "<" + c + ">"
            enc = port.encode(port.decode(json.dumps(obj, ensure_ascii=False).encode()))
            a = enc.index(b'"correlation_id":"<') + len(b'"correlation_id":"<')
            ids.append(enc[a:enc.index(b'>"', a)])
        _SPELL = dict(zip(chars, ids))
        assert _SPELL["\n"] == b"\\n" and _SPELL["\x01"] == b"\\u0001" and _SPELL['"'] == b'\\"'
    return _SPELL


def _spell(s: str) -> bytes:
    sp = _spellings()
    return b"".join(sp.get(c, c.encode()) for c in s)


UTF8 = ["é", "ß", "€", "東", "京", "😀", "ü"]
ASCII = "abcdefghijklmnopqrstuvwxyz0123456789_-:. ABCXYZ"


def _fill(rng, nbytes: int) -> str:
    return "".join(rng.choice(ASCII) for _ in range(nbytes))


def _keys(seed: int) -> list[bytes]:
    """raw contents of every length 0-96 and sparse lengths up to 300: plain ASCII, random mixes, and each escape and
    multi-byte character at every position of every length 0-96"""
    rng = random.Random(seed)
    sp = _spellings()
    specials = [sp[c].decode() for c in sp] + UTF8
    lengths = list(range(97)) + [100, 111, 127, 128, 129, 160, 191, 192, 200, 255, 256, 257, 299, 300]
    out = []
    for L in lengths:
        out.append(_fill(rng, L).encode())
        for _ in range(3):                       # random mixes of ASCII, escapes and UTF-8 filled up to L bytes exactly
            s = ""
            while len(s.encode()) < L:
                tok = rng.choice(specials) if rng.random() < 0.3 else rng.choice(ASCII)
                s += tok if len(s.encode()) + len(tok.encode()) <= L else rng.choice(ASCII)
            out.append(s.encode())
    for L in range(97):
        for p in range(L):                       # one special at every position, rotating through all of them
            tok = specials[(p * 7 + L) % len(specials)]
            if p + len(tok.encode()) > L:
                tok = sp["\\"].decode() if p + 2 <= L else rng.choice(ASCII)
            out.append((_fill(rng, p) + tok + _fill(rng, L - p - len(tok.encode()))).encode())
    assert {len(k) for k in out} >= set(range(97))
    return out


def _prd_window_offset(rec_abs: int, prime: int, key_off: int) -> int:
    """where the key starts in the PRd window after the reader read byte `prime` (ck_p2_refill)"""
    m = rec_abs & 15
    wb = (m + prime) & ~15
    wb = wb - 16 if wb >= 16 else 0
    return m + key_off - wb


def _key_records(seed: int):
    """records packed back to back, each holding one key: -> (bytes, offsets, [(record, off, len, prime)], keys)"""
    rng = random.Random(seed)
    keys = _keys(seed)
    junk = ASCII + "\\" * 16 + '"{}:,'           # around the keys: backslashes the 8-byte pass must not count as the key's
    recs, quads = [], []
    pos = 0
    for j, raw in enumerate(keys):
        kind = j % 4                  # 0: key mid-record; 1: key ends on the record's last byte; 2, 3: primed window
        pre = rng.randrange(0, 40) if kind < 2 else rng.randrange(72, 140)
        prefix = "".join(rng.choice(junk) for _ in range(pre)).encode()
        suffix = b"" if kind == 1 else ('"' + "".join(rng.choice(junk) for _ in range(rng.randrange(0, 24)))).encode()
        prime = 0xFFFFFFFF
        if kind >= 2:                 # the key starts 40-63 bytes into the window: it refills in the middle of the hash
            prime = rng.choice([x for x in range(pre) if 40 <= _prd_window_offset(pos, x, pre) < 64])
        recs.append(prefix + raw + suffix)
        quads.append((j, pre, len(raw), prime))
        pos += len(recs[-1])
    offs = np.zeros(len(recs) + 1, np.int64)
    offs[1:] = np.cumsum([len(r) for r in recs])
    starts = {(int(offs[q[0]]) + q[1]) % 16 for q in quads}
    assert starts == set(range(16))
    return b"".join(recs), offs, np.array(quads, np.uint32), keys


@pytest.fixture(scope="module")
def key_case():
    data, offs, quads, keys = _key_records(5)
    want = np.array([_murmur2(json.loads(b'"' + k + b'"').encode()) for k in keys], np.uint32)
    assert all(json.loads(b'"' + k + b'"').encode() == k for k in keys if b"\\" not in k)
    return data, offs, quads, keys, want


def _hash(dev, reader: int, data: bytes, offs, quads):
    import torch
    import devsim
    d_in = _cuda(_with_slack(np.frombuffer(data, np.uint8)))
    d_off, d_q = _cuda(offs), _cuda(quads.view(np.int32))
    n = len(quads)
    h = torch.zeros(n, dtype=torch.int32, device="cuda")
    reads = torch.zeros(n, dtype=torch.int32, device="cuda")
    devsim.check(dev.ck_dev_murmur2_key(reader, d_in.data_ptr(), d_off.data_ptr(), len(offs) - 1, d_q.data_ptr(), n,
                                        h.data_ptr(), reads.data_ptr()))
    return h.cpu().numpy().view(np.uint32), reads.cpu().numpy()


@pytest.mark.parametrize("reader", [0, 1], ids=["PRd", "GRd"])
def test_murmur2_key_matches_kafka_murmur2_of_unescaped_key(dev, key_case, reader):
    """all 32 bits of ck_murmur2_key against Kafka's murmur2 of the unescaped key, through the plan's window (PRd) and the
    route kernel's global loads (GRd)"""
    data, offs, quads, keys, want = key_case
    got, _ = _hash(dev, reader, data, offs, quads)
    bad = np.flatnonzero(got != want)
    assert bad.size == 0, [(keys[j], int(quads[j][3]) != 0xFFFFFFFF, hex(got[j]), hex(want[j])) for j in bad[:10]] + [bad.size]


def test_murmur2_key_decodes_only_keys_with_escapes(dev, key_case):
    """the 8-byte pass finds every backslash of the key and nothing past it: a key without an escape is hashed without a
    single byte read (the decoding pass), a key with one is decoded"""
    data, offs, quads, keys, want = key_case
    got, reads = _hash(dev, 2, data, offs, quads)
    assert (got == want).all()
    esc = np.array([b"\\" in k for k in keys])
    assert esc.sum() > 1000 and (~esc).sum() > 500
    bad = np.flatnonzero((reads > 0) != esc)
    assert bad.size == 0, [(keys[j], int(reads[j])) for j in bad[:10]] + [bad.size]
