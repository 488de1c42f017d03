"""numpy restatement of the dropout masks documented in include/fsb200.h (Philox4x32-10 and the two counter layouts). The
GPU dropout tests build every mask from here, independently of the library."""
import numpy as np

_M0, _M1, _W0, _W1 = 0xD2511F53, 0xCD9E8D57, 0x9E3779B9, 0xBB67AE85
_MASK = np.uint64(0xFFFFFFFF)


def philox4x32_10(ctr, key):
    """ctr: four uint32 arrays (broadcastable), key: (k0, k1) ints. Returns four uint32 arrays."""
    c0, c1, c2, c3 = (np.asarray(c, dtype=np.uint64) & _MASK for c in ctr)
    c0, c1, c2, c3 = np.broadcast_arrays(c0, c1, c2, c3)
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        p0 = c0 * np.uint64(_M0)
        p1 = c2 * np.uint64(_M1)
        hi0, lo0 = p0 >> np.uint64(32), p0 & _MASK
        hi1, lo1 = p1 >> np.uint64(32), p1 & _MASK
        c0, c1, c2, c3 = hi1 ^ c1 ^ np.uint64(k0), lo1, hi0 ^ c3 ^ np.uint64(k1), lo0
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return tuple(c.astype(np.uint32) for c in (c0, c1, c2, c3))


def threshold(p):
    """Drop when the 8-bit value is below this: floor(p * 256 + 0.5) in fp32."""
    return int(np.floor(np.float32(p) * np.float32(256.0) + np.float32(0.5)))


def p_eff(p):
    return threshold(p) / 256.0


def _key(seed):
    seed = int(seed) & 0xFFFFFFFFFFFFFFFF
    return seed & 0xFFFFFFFF, seed >> 32


def _stream(stream):
    s = int(stream) & 0xFFFFFFFFFFFFFFFF
    return s & 0xFFFFFFFF, s >> 32


def _bytes(words, word_idx, byte_idx):
    w = np.choose(word_idx, words)
    return (w >> (8 * byte_idx).astype(np.uint32)) & np.uint32(0xFF)


def hidden_keep(seed, stream, rows, cols, p):
    """Keep mask (bool [rows, cols]) of hidden dropout: counter (col / 16, row, stream lo, stream hi), byte col % 16."""
    r = np.arange(rows, dtype=np.uint64)[:, None]
    c = np.arange(cols, dtype=np.int64)[None, :]
    s_lo, s_hi = _stream(stream)
    words = philox4x32_10(((c >> 4).astype(np.uint64), r, s_lo, s_hi), _key(seed))
    words = [np.broadcast_to(w, (rows, cols)) for w in words]
    cb = np.broadcast_to(c & 15, (rows, cols))
    return _bytes(words, cb >> 2, cb & 3) >= threshold(p)


def attn_keep(seed, stream, batch, nheads, seq_q, seq_kv, p):
    """Keep mask (bool [batch, nheads, seq_q, seq_kv]) of attention dropout (layout in include/fsb200.h)."""
    q = np.arange(seq_q, dtype=np.int64)[:, None]
    k = np.arange(seq_kv, dtype=np.int64)[None, :]
    qa, qh, qs, qp = q >> 4, (q >> 3) & 1, (q >> 1) & 3, q & 1
    ka, kh, ks, kp = k >> 4, (k >> 3) & 1, (k >> 1) & 3, k & 1
    x0 = ((ka * 4 + ks) | ((qa * 4 + qs) << 16)).astype(np.uint64)
    word = np.broadcast_to(2 * qp + kp, (seq_q, seq_kv))
    byte = np.broadcast_to(2 * qh + kh, (seq_q, seq_kv))
    s_lo, s_hi = _stream(stream)
    out = np.empty((batch, nheads, seq_q, seq_kv), dtype=bool)
    for b in range(batch):
        for h in range(nheads):
            words = [np.broadcast_to(w, (seq_q, seq_kv)) for w in philox4x32_10((x0, b * nheads + h, s_lo, s_hi), _key(seed))]
            out[b, h] = _bytes(words, word, byte) >= threshold(p)
    return out
