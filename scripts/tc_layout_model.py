"""Address-level model of the Hopper tensor-core data path of csrc/attn_tc.cuh and csrc/conv_tc.cu, in numpy.

Shared memory is a byte array.  TMA with SWIZZLE_128B stores row r of a [rows][64 halfs] tile at r * 128 with its 16-byte
chunk c at chunk c ^ (r % 8); the conv producer writes its activation slots with the same formula as the kernel (soff).
wgmma reads operands through the same descriptor arithmetic as the kernels (start address + 32 B per 16-deep k-step of a
K-major operand, + 64 B for the lo halves, + 2048 B per k-step of an MN-major operand; 8-row groups 1024 B apart), and
thread fragments follow the PTX wgmma tables (accumulator d[j] of lane l in warp w: row 16 w + l / 4 + 8 ((j / 2) % 2),
column 8 (j / 4) + 2 (l % 4) + j % 2; register A operand = the accumulator fragment of 16 columns re-packed as fp16).
Under this model the kernels' addressing must reproduce attention and convolution exactly as the reference formulas.
"""
import numpy as np


def swz(row, byte):                      # byte offset of (row, byte within the 128 B row) in a SWIZZLE_128B tile
    return row * 128 + (((byte // 16) ^ (row % 8)) * 16) + byte % 16


def tma_store(buf, base, tile):          # tile: [rows][64] fp16
    raw = tile.astype(np.float16).view(np.uint8).reshape(tile.shape[0], 128)
    for r in range(tile.shape[0]):
        for b in range(128):
            buf[base + swz(r, b)] = raw[r, b]


def half_at(buf, addr):
    return buf[addr:addr + 2].view(np.float16)[0]


def read_kmajor(buf, start, rows):
    """16-deep k-step of a K-major operand at descriptor start address `start`: [rows][16]."""
    out = np.zeros((rows, 16), np.float32)
    for i in range(rows):
        for k in range(16):
            off = start + (i // 8) * 1024 + (i % 8) * 128 + 2 * k    # unswizzled address the descriptor names
            row_base = off - (off % 128)
            byte = off % 128
            r = (row_base // 128) % 8                                 # swizzle uses address bits [7, 10)
            out[i, k] = half_at(buf, row_base + (((byte // 16) ^ r) * 16) + byte % 16)
    return out


def read_mnmajor(buf, start, n):
    """16-deep k-step of an MN-major operand (rows = K index, 64 halfs of N per row): [16][n]."""
    out = np.zeros((16, n), np.float32)
    for k in range(16):
        for j in range(n):
            off = start + k * 128 + 2 * j
            row_base = off - (off % 128)
            byte = off % 128
            r = (row_base // 128) % 8
            out[k, j] = half_at(buf, row_base + (((byte // 16) ^ r) * 16) + byte % 16)
    return out


def frag_coords(n):
    """(warp, lane, j) -> (row, col) of the m64nN fp32 accumulator."""
    for w in range(4):
        for l in range(32):
            for j in range(n // 2):
                yield w, l, j, 16 * w + l // 4 + 8 * ((j // 2) % 2), 8 * (j // 4) + 2 * (l % 4) + j % 2


def a_from_acc(acc_regs, kk):
    """Register A operand of k-step kk as the kernel packs it: a[0..3] = d[8kk + 0..7] in pairs -> [64][16] matrix."""
    A = np.zeros((64, 16), np.float32)
    for w in range(4):
        for l in range(32):
            r0, c = 16 * w + l // 4, 2 * (l % 4)
            d = acc_regs[w][l]
            for t, (rr, cc) in enumerate(((r0, c), (r0 + 8, c), (r0, c + 8), (r0 + 8, c + 8))):
                A[rr, cc] = np.float16(d[8 * kk + 2 * t])
                A[rr, cc + 1] = np.float16(d[8 * kk + 2 * t + 1])
    return A


def split(x):
    hi = x.astype(np.float16)
    lo = (x - hi.astype(np.float32)).astype(np.float16)
    return hi, lo


def reference(Q, K, V, T):
    s = (Q / T) @ K.T
    p = np.exp(s - s.max(1, keepdims=True))
    return (p / p.sum(1, keepdims=True)) @ V


def model_attention(Q, K, V, T, qc=1, bk=64):
    """One warpgroup (64 queries) of attn_tc_kernel in exact mode over all keys: Q [64][32 qc], K [Tk][32 qc], V [Tk][32]."""
    Tk = K.shape[0]
    Qs = (Q / np.float32(T)).astype(np.float32)
    buf = np.zeros(qc * 64 * 128 + qc * bk * 128 + bk * 128, np.uint8)
    for c in range(qc):                                   # Q chunks [hi | lo]
        hi, lo = split(Qs[:, 32 * c:32 * c + 32])
        tma_store(buf, c * 64 * 128, np.concatenate([hi, lo], 1))
    kbase, vbase = qc * 64 * 128, qc * 64 * 128 + qc * bk * 128
    m = np.full(64, -np.inf, np.float32)
    lsum = np.zeros(64, np.float32)
    O = np.zeros((64, 64), np.float32)
    for k0 in range(0, Tk, bk):
        Kt = np.zeros((bk, 32 * qc), np.float32)
        Vt = np.zeros((bk, 32), np.float32)
        live = min(bk, Tk - k0)
        Kt[:live], Vt[:live] = K[k0:k0 + live], V[k0:k0 + live]
        for c in range(qc):
            hi, lo = split(Kt[:, 32 * c:32 * c + 32])
            tma_store(buf, kbase + c * bk * 128, np.concatenate([hi, lo], 1))
        vh, vl = split(Vt)
        tma_store(buf, vbase, np.concatenate([vh, vl], 1))
        S = np.zeros((64, bk), np.float32)
        for c in range(qc):
            q0, kq = c * 64 * 128, kbase + c * bk * 128
            for ks in range(2):                             # descriptor +2 (32 B) per k-step, +4 (64 B) for lo
                Qh, Ql = read_kmajor(buf, q0 + 32 * ks, 64), read_kmajor(buf, q0 + 64 + 32 * ks, 64)
                Kh, Kl = read_kmajor(buf, kq + 32 * ks, bk), read_kmajor(buf, kq + 64 + 32 * ks, bk)
                S += Qh @ Kh.T + Ql @ Kh.T + Qh @ Kl.T
        S[:, live:] = -np.inf
        regs = [[np.zeros(bk // 2, np.float32) for _ in range(32)] for _ in range(4)]
        for w, l, j, r, col in frag_coords(bk):
            regs[w][l][j] = S[r, col]
        mx = np.maximum(m, S.max(1))
        f = np.exp(m - mx)
        lsum *= f
        O *= f[:, None]
        m = mx
        P = np.exp(S - m[:, None]).astype(np.float32)
        lsum += P.sum(1)
        for w, l, j, r, col in frag_coords(bk):
            regs[w][l][j] = P[r, col]
        lo_regs = [[np.zeros(bk // 2, np.float32) for _ in range(32)] for _ in range(4)]
        for w in range(4):
            for l in range(32):
                lo_regs[w][l] = regs[w][l] - regs[w][l].astype(np.float16).astype(np.float32)
        for kk in range(bk // 16):                         # V MN-major: +128 (2048 B) per k-step
            Vk = read_mnmajor(buf, vbase + 2048 * kk, 64)
            O += a_from_acc(regs, kk) @ Vk + a_from_acc(lo_regs, kk) @ Vk
    return (O[:, :32] + O[:, 32:]) / lsum[:, None]


def model_conv_a_tile(X):
    """conv_tc.cu: for half chunk `part`, producer thread p (q = p & 15, rsub = p >> 4) stores rows part*64 + i*8 + rsub,
    16-byte segment q, hi half at soff + part*8192 + i*1024; consumer warpgroup wg's wgmma reads rows [wg*64, +64) K-major
    from start + wg*8192 + 32 ks.  X: [128][64] fp32 -> the [128][64] matrix (hi halves) the MMAs see."""
    buf = np.zeros(128 * 128, np.uint8)
    hi = X.astype(np.float16)
    for part in range(2):
        for p in range(128):
            q, rsub = p & 15, p >> 4
            soff = (part * 64 + rsub) * 128 + (((q >> 1) ^ rsub) << 4) + ((q & 1) << 3)
            for i in range(8):
                row = part * 64 + i * 8 + rsub
                buf[soff + i * 1024: soff + i * 1024 + 8] = hi[row, 4 * q:4 * q + 4].view(np.uint8)
    out = np.zeros((128, 64), np.float32)
    for wg in range(2):
        for ks in range(4):
            out[wg * 64:wg * 64 + 64, 16 * ks:16 * ks + 16] = read_kmajor(buf, wg * 8192 + 32 * ks, 64)
    return out
