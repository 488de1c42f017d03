"""numpy restatement of the dropout masks documented in include/fsb200.h (Philox4x32-10 and the two counter layouts). The
GPU dropout tests build every mask from here, independently of the library."""
import numpy as np
import torch

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


# ------------------------------------------------------------------------------------------------------ torch port
# The same masks computed with torch int64 tensors on any device, for the bench-sized masks the launch census checks (a
# MegatronBERT attention mask has 2.7e8 elements). 32-bit words live in int64 tensors; the 32 x 32-bit products are formed
# from 16-bit halves of the constant, so no intermediate leaves int64. tests/test_launch_refs_cpu.py pins it to the numpy
# version above, bit for bit.
def _mulhilo_t(a, m):
    """(hi, lo) 32-bit words of a * m for int64 tensors a in [0, 2^32) and a 32-bit constant m."""
    lo_part, hi_part = a * (m & 0xFFFF), a * (m >> 16)            # each < 2^48
    t = lo_part + ((hi_part & 0xFFFF) << 16)                      # a * m = t + (hi_part >> 16) 2^32
    return (t >> 32) + (hi_part >> 16), t & 0xFFFFFFFF


def philox4x32_10_t(ctr, key):
    """ctr: four int64 tensors (or ints) holding uint32 values, broadcastable; key (k0, k1). Returns four int64 tensors."""
    dev = next((c.device for c in ctr if isinstance(c, torch.Tensor)), torch.device("cpu"))
    c0, c1, c2, c3 = torch.broadcast_tensors(*(torch.as_tensor(c, dtype=torch.int64, device=dev) for c in ctr))
    k0, k1 = int(key[0]) & 0xFFFFFFFF, int(key[1]) & 0xFFFFFFFF
    for _ in range(10):
        hi0, lo0 = _mulhilo_t(c0, _M0)
        hi1, lo1 = _mulhilo_t(c2, _M1)
        c0, c1, c2, c3 = hi1 ^ c1 ^ k0, lo1, hi0 ^ c3 ^ k1, lo0
        k0, k1 = (k0 + _W0) & 0xFFFFFFFF, (k1 + _W1) & 0xFFFFFFFF
    return c0, c1, c2, c3


def _bytes_t(words):
    """[..., 4 words] -> [..., 4 words, 4 bytes] of 8-bit values."""
    w = torch.stack(words, -1)
    return torch.stack([(w >> (8 * b)) & 0xFF for b in range(4)], -1)


def hidden_keep_t(seed, stream, rows, cols, p, device="cpu"):
    """hidden_keep for the rows in `rows` (a range) on `device`: bool [len(rows), cols]."""
    r = torch.arange(rows.start, rows.stop, dtype=torch.int64, device=device)[:, None]
    c16 = torch.arange((cols + 15) // 16, dtype=torch.int64, device=device)[None, :]
    s_lo, s_hi = _stream(stream)
    words = philox4x32_10_t((c16, r, s_lo, s_hi), _key(seed))
    by = _bytes_t(words)                                           # [rows, col16, word, byte]: column 16 c16 + 4 word + byte
    return by.reshape(r.shape[0], -1)[:, :cols] >= threshold(p)


def attn_keep_t(seed, stream, batches, nheads, seq_q, seq_kv, p, device="cpu"):
    """attn_keep for the batch rows in `batches` (a range) on `device`: bool [len(batches), nheads, seq_q, seq_kv]. One
    Philox call per 4 x 4 block (qa, qs) x (ka, ks); word 2 qp + kp, byte 2 qh + kh."""
    QA, KA = (seq_q + 15) // 16, (seq_kv + 15) // 16
    bh = (torch.arange(batches.start, batches.stop, dtype=torch.int64, device=device)[:, None] * nheads
          + torch.arange(nheads, dtype=torch.int64, device=device)[None, :]).reshape(-1, 1, 1)
    qc = torch.arange(4 * QA, dtype=torch.int64, device=device).view(1, -1, 1)    # 4 qa + qs
    kc = torch.arange(4 * KA, dtype=torch.int64, device=device).view(1, 1, -1)    # 4 ka + ks
    s_lo, s_hi = _stream(stream)
    words = philox4x32_10_t((kc | (qc << 16), bh, s_lo, s_hi), _key(seed))
    by = _bytes_t(words)                                           # [bh, 4 qa + qs, 4 ka + ks, 2 qp + kp, 2 qh + kh]
    nb = bh.shape[0]
    by = by.view(nb, QA, 4, KA, 4, 2, 2, 2, 2)                     # [bh, qa, qs, ka, ks, qp, kp, qh, kh]
    by = by.permute(0, 1, 7, 2, 5, 3, 8, 4, 6)                     # [bh, qa, qh, qs, qp, ka, kh, ks, kp]
    keep = by.reshape(nb, 16 * QA, 16 * KA)[:, :seq_q, :seq_kv] >= threshold(p)
    return keep.view(len(batches), nheads, seq_q, seq_kv)
