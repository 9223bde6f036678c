"""TEST INFRASTRUCTURE (oracle): numpy restatement of the *stream format* - the one-time re-layout of a
GEMM-layout AWQ linear (awq/modules/linear/gemm.py:135-158: qweight [K, N/8] i32, qzeros [K/G, N/8] i32, scales
[K/G, N] f16) that the decode-program kernel streams (autoawq_b200/csrc/program_stream.cuh; the reference's
precedent for a post-load re-layout is awq/modules/linear/exllama.py:66-79).  Only tests may import this.

The format (per linear), all little-endian:

  * columns are taken in SETS of 16 (one m16n8k16 MMA tile: A rows = 16 output columns); set s holds the columns
        mode 0 (plain):      lo[g] = 16 s + g,  hi[g] = 16 s + 8 + g            g = 0..7
        mode 1 (gate | up):  lo[g] =  8 s + g,  hi[g] = N/2 + 8 s + g           (SiLU*mul pairs share a lane)
  * K is cut in UNITS of UK = min(G, 128) rows; one unit of one set is contiguous:
        F = UK / 16 fragments of 128 bytes  +  48 bytes of group constants  =  F * 128 + 48 bytes
    and the buffer is set-major: byte offset of unit j of set s = (s * (K / UK) + j) * unit_bytes.
  * fragment f of a unit covers rows k0 = unit_k0 + 16 f .. + 15; its 32 words are the A fragments of the 32
    lanes of a warp, lane = 4 g + tig:  word = sum_i nib_i << 4 i  with
        nib0 = q[k0 + 2 tig    , lo[g]]   nib4 = q[k0 + 2 tig + 1, lo[g]]      -> a0 = (w      & 0x000f000f) | 0x6400
        nib1 = q[k0 + 2 tig    , hi[g]]   nib5 = q[k0 + 2 tig + 1, hi[g]]      -> a1 = (w      & 0x00f000f0) | 0x6400
        nib2 = q[k0 + 2 tig + 8, lo[g]]   nib6 = q[k0 + 2 tig + 9, lo[g]]      -> a2 = (w >> 8 & 0x000f000f) | 0x6400
        nib3 = q[k0 + 2 tig + 8, hi[g]]   nib7 = q[k0 + 2 tig + 9, hi[g]]      -> a3 = (w >> 8 & 0x00f000f0) | 0x6400
    i.e. lo columns come out as the fp16 pair (1024 + q), hi columns as (1024 + 16 q) - the raw-code trick of
    the persistent GEMV (csrc/gemv.cu); fragments are stored in QUADS for F >= 4 ([F/4][lane][4 words], one
    LDS.128 per lane = 4 MMAs) and as one pair for F = 2 ([lane][2 words]).
  * group constants (group of the unit's rows): 8 x (fp16 scale of lo[g], fp16 scale of hi[g]) = 32 bytes, then 8
    bytes (zero of lo[g]) | (zero of hi[g]) << 4, then 8 bytes of zero padding.
"""
import numpy as np

REV = np.array([0, 4, 1, 5, 2, 6, 3, 7])  # nibble position of column j within a GEMM-layout word (AWQ_REVERSE_ORDER)


def unit_k(G):
    return min(G, 128)


def unit_bytes(G):
    return unit_k(G) // 16 * 128 + 48


def stream_bytes(K, N, G):
    return (N // 16) * (K // unit_k(G)) * unit_bytes(G)


def set_columns(N, mode):
    """[S, 16] original column of (set, row of the MMA tile): rows 0..7 = lo[g], rows 8..15 = hi[g]."""
    S = N // 16
    s = np.arange(S)[:, None]
    g = np.arange(8)[None, :]
    if mode == 0:
        lo, hi = 16 * s + g, 16 * s + 8 + g
    else:
        lo, hi = 8 * s + g, N // 2 + 8 * s + g
    return np.concatenate([lo, hi], axis=1)


def unpack_gemm_ints(qweight, qzeros):
    """Canonical integers from the GEMM layout: iw [K, N], iz [K/G, N] (awq/utils/packing_utils.py:8-43)."""
    sh = (4 * REV).astype(np.uint32)
    qw = qweight.view(np.uint32)[:, :, None] >> sh[None, None, :]
    qz = qzeros.view(np.uint32)[:, :, None] >> sh[None, None, :]
    return (qw & 0xF).astype(np.uint8).reshape(qweight.shape[0], -1), (qz & 0xF).astype(np.uint8).reshape(qzeros.shape[0], -1)


def pack_stream(qweight, qzeros, scales, G, mode=0):
    """GEMM-layout tensors -> stream buffer (uint8 array).  Requires N % 16 == 0, K % UK == 0, G % UK == 0."""
    K, N = qweight.shape[0], qweight.shape[1] * 8
    UK = unit_k(G)
    assert N % 16 == 0 and K % UK == 0 and G % UK == 0 and UK % 32 == 0
    if mode == 1:
        assert N % 16 == 0 and (N // 2) % 8 == 0
    F, NU, S, UB = UK // 16, K // UK, N // 16, unit_bytes(G)
    iw, iz = unpack_gemm_ints(qweight, qzeros)
    cols = set_columns(N, mode)                    # [S, 16]
    out = np.zeros((S, NU, UB), dtype=np.uint8)
    # q[s, r, k] for tile row r (0..15)
    q = iw[:, cols].transpose(1, 2, 0).astype(np.uint32)          # [S, 16, K]
    q = q.reshape(S, 16, NU, F, 16)                               # k = (unit, frag, kk)
    g = np.arange(8)
    words = np.zeros((S, NU, F, 8, 4), dtype=np.uint32)           # [.., g, tig]
    for tig in range(4):
        k = 2 * tig
        lo, hi = q[:, 0:8], q[:, 8:16]                            # [S, 8, NU, F, 16]
        w = (lo[..., k] | hi[..., k] << 4 | lo[..., k + 8] << 8 | hi[..., k + 8] << 12 |
             lo[..., k + 1] << 16 | hi[..., k + 1] << 20 | lo[..., k + 9] << 24 | hi[..., k + 9] << 28)
        words[..., tig] = w.transpose(0, 2, 3, 1)                 # [S, NU, F, 8]
    words = words.reshape(S, NU, F, 32)                           # lane = 4 g + tig
    if F >= 4:
        frag = words.reshape(S, NU, F // 4, 4, 32).transpose(0, 1, 2, 4, 3)   # [quad][lane][4]
    else:
        frag = words.transpose(0, 1, 3, 2)                                     # [lane][2]
    out[:, :, : F * 128] = np.ascontiguousarray(frag).reshape(S, NU, F * 32).view(np.uint8).reshape(S, NU, F * 128)
    # group constants
    grp = (np.arange(NU) * UK) // G                               # group of each unit
    sc = scales[grp][:, cols]                                     # [NU, S, 16] fp16
    sc = sc.transpose(1, 0, 2)                                    # [S, NU, 16]
    sc2 = np.stack([sc[..., 0:8], sc[..., 8:16]], axis=-1)        # [S, NU, 8, 2] = (lo[g], hi[g])
    out[:, :, F * 128: F * 128 + 32] = np.ascontiguousarray(sc2).view(np.uint8).reshape(S, NU, 32)
    z = iz[grp][:, cols].transpose(1, 0, 2)                       # [S, NU, 16]
    out[:, :, F * 128 + 32: F * 128 + 40] = (z[..., 0:8] | (z[..., 8:16] << 4)).astype(np.uint8)
    return out.reshape(-1)


def simulate_gemv(stream, K, N, G, x, mode=0):
    """y[N] (float64) from the stream buffer and x[K] (fp16), following the kernel's arithmetic contract: per unit
    S = sum_k x_k * (1024 + c q) exactly, y += s * (S - (1024 + c z) * X) / c.  Used to pin the format itself
    (which nibble sits where) independently of the CUDA code."""
    UK = unit_k(G)
    F, NU, S, UB = UK // 16, K // UK, N // 16, unit_bytes(G)
    buf = np.asarray(stream, dtype=np.uint8).reshape(S, NU, UB)
    cols = set_columns(N, mode)
    y = np.zeros(N, dtype=np.float64)
    xf = np.asarray(x, dtype=np.float64).reshape(NU, F, 16)
    for s in range(S):
        for j in range(NU):
            u = buf[s, j]
            words = u[: F * 128].view(np.uint32)
            if F >= 4:
                words = words.reshape(F // 4, 32, 4).transpose(0, 2, 1).reshape(F, 32)
            else:
                words = words.reshape(32, F).T
            sc = u[F * 128: F * 128 + 32].view(np.float16).astype(np.float64).reshape(8, 2)
            zb = u[F * 128 + 32: F * 128 + 40]
            S_lo, S_hi = np.zeros(8), np.zeros(8)
            X = xf[j].sum()
            for f in range(F):
                for lane in range(32):
                    g, tig = lane >> 2, lane & 3
                    w = int(words[f, lane])
                    nib = [(w >> (4 * i)) & 0xF for i in range(8)]
                    xk = xf[j, f]
                    S_lo[g] += (xk[2 * tig] * (1024 + nib[0]) + xk[2 * tig + 1] * (1024 + nib[4]) +
                                xk[2 * tig + 8] * (1024 + nib[2]) + xk[2 * tig + 9] * (1024 + nib[6]))
                    S_hi[g] += (xk[2 * tig] * (1024 + 16 * nib[1]) + xk[2 * tig + 1] * (1024 + 16 * nib[5]) +
                                xk[2 * tig + 8] * (1024 + 16 * nib[3]) + xk[2 * tig + 9] * (1024 + 16 * nib[7]))
            for g in range(8):
                zl, zh = int(zb[g]) & 0xF, int(zb[g]) >> 4
                y[cols[s, g]] += sc[g, 0] * (S_lo[g] - (1024 + zl) * X)
                y[cols[s, 8 + g]] += sc[g, 1] / 16 * (S_hi[g] - (1024 + 16 * zh) * X)
    return y
