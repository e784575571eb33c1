"""Plain references the tests share (TEST INFRASTRUCTURE, CPU only): the local distance, the banded, full-matrix,
any-rate and path DPs, the decision rules, DTW barycentre averaging, the connected-word and grammar helpers, the
long-form VAD transcribed from VAD.C, and the host's launch plan of the connected-word calls. Each is written from its
definition and shares no code with oracle/sr_oracle.c or tests/oracle_ext, so that a mistake common to a kernel and its
oracle still fails a test. Bare asserts here are not rewritten by pytest, so each one carries a message."""
import os

import numpy as np

import oracle_bind as ob
import sr_b200

DIS_ERR = NULL = 0xFFFFFFFF
MAX_FRM = 119
NTHREADS = max(1, min(16, os.cpu_count() or 1))
STRIDE = ob.FTR_DTYPE.itemsize
# rows with get_dis(MAX_A, MAX_B) = 65 536, the largest local distance: 65535^2 + 362^2 = 2^32 - 27 rounds to 2^32 in
# float32. A pair of such constant feature sets has D(I-1,M-1) = max(I,M) * 65 536, the largest result any pair can have
MAX_A = np.array([32767, 362] + [0] * 10, np.int16)
MAX_B = np.array([-32768, 0] + [0] * 10, np.int16)


# ---- the local distance and the template DPs -------------------------------------------------------------------------
def get_dis(a, b):
    """get_dis (DTW.C:45-62) of two rows: u32-wrapped sum of squares, float32 square root, truncated"""
    s = int(sum((int(x) - int(y)) ** 2 for x, y in zip(a, b))) & 0xFFFFFFFF
    return int(np.sqrt(np.float32(s), dtype=np.float32))


def dist_matrix(a, b):
    """get_dis (DTW.C:45-62) of every row of a [I,12] against every row of b [M,12]: the sum of the 12 squared differences
    wrapped to u32, converted to float32, IEEE square root in float32, truncated"""
    dif = a.astype(np.int64)[:, None, :] - b.astype(np.int64)[None, :, :]
    s = ((dif * dif).sum(axis=2) & 0xFFFFFFFF).astype(np.uint32)
    return np.sqrt(s.astype(np.float32)).astype(np.uint32).astype(np.int64)


def guard_rejects(I, M):
    """the 2:1 length guard of dtw (DTW.C:133), and the empty sets that have no cell"""
    return I == 0 or M == 0 or I > 2 * M or M > 2 * I


def band_dp_ref(fin, fmdl, r, with_d=False):
    """D(i,j) = d(i,j) + min(D(i-1,j), D(i,j-1), D(i-1,j-1)), D(0,0) = d(0,0), over the whole I x M matrix in exact
    integers, +inf outside the band |j - floor(i*M/I)| <= r; the result is D(I-1,M-1) // (I+M), dis_err when that cell is
    unreachable. with_d: (result, D(I-1,M-1))"""
    I, M = len(fin), len(fmdl)
    if guard_rejects(I, M):
        return (DIS_ERR, None) if with_d else DIS_ERR
    d = dist_matrix(fin, fmdl).tolist()
    inf = float("inf")
    D = [[inf] * M for _ in range(I)]
    for i in range(I):
        c = i * M // I
        for j in range(M):
            if abs(j - c) > r:
                continue
            if i == 0 and j == 0:
                best = 0
            else:
                best = min(D[i - 1][j] if i else inf, D[i][j - 1] if j else inf, D[i - 1][j - 1] if i and j else inf)
            D[i][j] = best + d[i][j]
    end = D[I - 1][M - 1]
    res = DIS_ERR if end == inf else int(end) // (I + M)
    return (res, None if end == inf else int(end)) if with_d else res


def full_dp_ref(fin, fmdl):
    """textbook DTW over the full matrix (no band), same local distance, guard and normalisation"""
    I, M = len(fin), len(fmdl)
    if guard_rejects(I, M):
        return DIS_ERR
    d = dist_matrix(fin, fmdl)
    D = np.zeros((I, M), np.int64)
    for i in range(I):
        for j in range(M):
            prev = [D[i - 1, j]] if i else []
            prev += [D[i, j - 1]] if j else []
            prev += [D[i - 1, j - 1]] if i and j else []
            D[i, j] = d[i, j] + (min(prev) if prev else 0)
    return int(D[I - 1, M - 1]) // (I + M)


def rate_ref(x, y, r):
    """D(I-1, M-1) of the band DP, cell by cell, without any length guard, or None when unreachable"""
    I, M = len(x), len(y)
    D = {}
    for i in range(I):
        for j in range(M):
            if abs(j - (i * M) // I) > r:
                continue
            prev = [D[c] for c in ((i - 1, j), (i, j - 1), (i - 1, j - 1)) if c in D]
            if i == j == 0:
                prev = [0]
            if prev:
                D[i, j] = min(prev) + get_dis(x[i], y[j])
    return D.get((I - 1, M - 1))


def want_best(score):
    """(best_idx, best_dis) of each score row: the first of the minima"""
    T = score.shape[1]
    key = (score.astype(np.uint64) << np.uint64(32)) | np.arange(T, dtype=np.uint64)[None, :]
    k = key.min(axis=1)
    return (k & np.uint64(0xFFFFFFFF)).astype(np.uint32), (k >> np.uint64(32)).astype(np.uint32)


def decide(score, k=0, q=0):
    """(best_idx, best_dis, cmd, reject) of each row of score [N][T] under SR_DTW_KNN(k) | SR_DTW_REJECT(q); k = 0 is the
    nearest-slot decision of main.c:276-292, and KNN(1) | REJECT(q) the margin rule"""
    score = np.asarray(score, np.uint32)
    N, T = score.shape
    C = (T + 3) // 4
    s = np.full((N, 4 * C), DIS_ERR, np.uint64)
    s[:, :T] = score
    s = s.reshape(N, C, 4)
    n = (s != DIS_ERR).sum(axis=2)
    m = np.minimum(max(k, 1), n)
    srt = np.sort(s, axis=2)                                             # SR_DIS_ERR last
    take = np.arange(4)[None, None, :] < m[:, :, None]
    e = np.where(m > 0, np.where(take, srt, 0).sum(axis=2) // np.maximum(m, 1), DIS_ERR).astype(np.uint64)
    slot = np.arange(C)[None, :] * 4 + np.argmin(s, axis=2)              # first of the command's minima
    key = (e << np.uint64(32)) | np.where(m > 0, slot, 0).astype(np.uint64)
    c1 = np.argmin(key, axis=1)
    k1 = key[np.arange(N), c1]
    idx, d1 = (k1 & np.uint64(DIS_ERR)).astype(np.uint32), k1 >> np.uint64(32)
    others = np.where(np.arange(C)[None, :] == c1[:, None], np.uint64(DIS_ERR), e)
    d2 = others.min(axis=1, initial=DIS_ERR)
    rej = (q > 0) & (d2 != DIS_ERR) & (np.uint64(1000) * (d2 - d1) < np.uint64(q) * d1)
    return idx, d1.astype(np.uint32), idx // 4, rej


# ---- paths and averaging ---------------------------------------------------------------------------------------------
def band_matrix(fin, fmdl, r):
    """the whole I x M matrix D(i, j) = d(i, j) + min(D(i-1, j-1), D(i, j-1), D(i-1, j)), D(0, 0) = d(0, 0), in exact
    integers (lists of lists), +inf outside the band |j - floor(i*M/I)| <= r and where unreachable; no length guard"""
    I, M = len(fin), len(fmdl)
    d = dist_matrix(fin, fmdl).tolist()
    inf = float("inf")
    D = [[inf] * M for _ in range(I)]
    for i in range(I):
        c = i * M // I
        for j in range(max(0, c - r), min(M - 1, c + r) + 1):
            if i == 0 and j == 0:
                D[i][j] = d[0][0]
                continue
            best = min(D[i - 1][j - 1] if i and j else inf, D[i][j - 1] if j else inf, D[i - 1][j] if i else inf)
            if best != inf:
                D[i][j] = best + d[i][j]
    return D


def band_path_ref(fin, fmdl, r):
    """(score, path, D(I-1,M-1)): band_matrix, then the trace-back from (I-1, M-1): the neighbour with the smallest D, ties
    to the diagonal, then (i, j-1), then (i-1, j). Rejected pairs: (DIS_ERR, [], None)"""
    I, M = len(fin), len(fmdl)
    if guard_rejects(I, M) or I > MAX_FRM or M > MAX_FRM:
        return DIS_ERR, [], None
    D = band_matrix(fin, fmdl, r)
    inf = float("inf")
    end = D[I - 1][M - 1]
    if end == inf:
        return DIS_ERR, [], None
    i, j, path = I - 1, M - 1, [(I - 1, M - 1)]
    while (i, j) != (0, 0):
        cand = [(D[i - 1][j - 1] if i and j else inf, 0), (D[i][j - 1] if j else inf, 1), (D[i - 1][j] if i else inf, 2)]
        k = min(cand)[1]                     # smallest D, then the lowest rank: diagonal, (i, j-1), (i-1, j)
        i, j = (i - 1, j - 1) if k == 0 else (i, j - 1) if k == 1 else (i - 1, j)
        path.append((i, j))
    return int(end) // (I + M), path[::-1], int(end)


def slot_rows(slot):
    """(save_sign, frm_num, rows [frm_num, 12]) of a bank slot (rows only when frm_num <= 119)"""
    f = slot[:STRIDE].view(ob.FTR_DTYPE)[0]
    n = int(f["frm_num"])
    return int(f["save_sign"]), n, (f["mfcc_dat"][: n * 12].reshape(n, 12).astype(np.int64) if n <= MAX_FRM else None)


def average_ref(bank, slot_stride, K, r, iters, ranges=None):
    """sr_average_bank from its definition: (bank_out, score [G, K], anchor [G]). ranges: a list that receives, per group
    with members and iters >= 1, the (lo, hi) per template cell of the frames the last update averaged"""
    bank = np.asarray(bank, np.uint8).reshape(-1, slot_stride)
    G = bank.shape[0] // K
    out = np.full_like(bank, 0xFF)
    score, anchor = np.full((G, K), DIS_ERR, np.uint32), np.full(G, 0xFFFFFFFF, np.uint32)
    for g in range(G):
        rows = {}
        for k in range(K):
            sign, n, x = slot_rows(bank[g * K + k])
            if sign == sr_b200.SAVE_MASK and 1 <= n <= MAX_FRM:
                rows[k] = x
        if not rows:
            continue
        S = {(l, k): band_path_ref(rows[l], rows[k], r)[0] for l in rows for k in rows if l != k}
        a = min(rows, key=lambda k: (sum(S[l, k] for l in rows if l != k), k))
        C = rows[a].copy()
        for _ in range(iters):
            tot, cnt = np.zeros_like(C), np.zeros(len(C), np.int64)
            lo, hi = np.full(C.shape, 1 << 20), np.full(C.shape, -(1 << 20))
            for l, x in rows.items():
                s, path, _ = band_path_ref(x, C, r)
                if s == DIS_ERR:
                    continue
                for i, j in path:
                    tot[j] += x[i]
                    cnt[j] += 1
                    lo[j], hi[j] = np.minimum(lo[j], x[i]), np.maximum(hi[j], x[i])
            if cnt.any():
                C = np.sign(tot) * (np.abs(tot) // cnt[:, None])         # C division truncates toward zero
                if ranges is not None:
                    ranges.append((g, lo, hi, C.copy()))
        M = len(C)
        out[g * K, :4] = np.frombuffer(np.array([sr_b200.SAVE_MASK, M], np.uint16).tobytes(), np.uint8)
        out[g * K, 4:4 + 24 * M] = np.frombuffer(C.astype(np.int16).tobytes(), np.uint8)
        for k, x in rows.items():
            score[g, k] = band_path_ref(x, C, r)[0]
        anchor[g] = a
    return out, score, anchor


# ---- connected words and grammars ------------------------------------------------------------------------------------
def bank_members(bank, n_slot, stride):
    """{slot: rows [M, 12]} of the members: save_sign == SR_SAVE_MASK and 1 <= frm_num <= 119"""
    out = {}
    for t in range(n_slot):
        sign, n = np.frombuffer(bank[t, :4].tobytes(), np.uint16)
        if sign == sr_b200.SAVE_MASK and 1 <= n <= MAX_FRM:
            out[t] = bank[t, 4:4 + 24 * int(n)].view(np.int16).reshape(int(n), 12).astype(np.int64)
    return out


def dtw_full(a, b):
    """unnormalised DTW over the full matrix, no 2:1 guard: D(I-1, M-1)"""
    d = dist_matrix(a, b)
    I, M = d.shape
    D = np.zeros((I, M), np.int64)
    for i in range(I):
        for j in range(M):
            prev = [D[i - 1, j]] if i else []
            prev += [D[i, j - 1]] if j else []
            prev += [D[i - 1, j - 1]] if i and j else []
            D[i, j] = d[i, j] + (min(prev) if prev else 0)
    return int(D[I - 1, M - 1])


def copies_of(grammar, mem):
    """[(state, slot, src mask)] state-major, then by slot"""
    S, _, arcs = grammar
    out = []
    for s in range(S):
        for t in sorted(mem):
            src = 0
            for a, b, m in arcs:
                if b == s and (m >> (t // 4)) & 1:
                    src |= 1 << a
            if src:
                out.append((s, t, src))
    return out


def accepts(grammar, cmds):
    """the grammar accepts the command sequence"""
    S, F, arcs = grammar
    cur = {0}
    for c in cmds:
        cur = {b for a, b, m in arcs if a in cur and (m >> c) & 1}
    return any(F >> s & 1 for s in cur)


# ---- the definition of the VAD, transcribed: VAD.C:97-218, u32 length ----------------------------------------------
def vad_frames(vc, n, atap):
    """the per-frame arithmetic of VAD.C:112-157 over the first n samples: (frm_sum, frm_zero, last_sig entering the
    frame), one int64 array each with one entry per frame i = 80k < n - 160. last_sig is never reset (VAD.C:99), so the
    frame enters with the class of the last out-of-band sample among samples <= 80k + 78: the previous frame scanned
    them."""
    mid, n_thl = int(atap["mid_val"]), int(atap["n_thl"])
    a_thl, b_thl = (mid + n_thl) & 0xFFFFFFFF, (mid - n_thl) & 0xFFFFFFFF       # VAD.C:112-113 (u32)
    vc = [int(v) for v in vc[:n]]
    sums, zeros, entry = [], [], []
    last_sig, i = 0, 0
    while n > 160 and i < n - 160:                                               # VAD.C:121
        entry.append(last_sig)
        sums.append(sum(abs(vc[i + h] - mid) for h in range(160)))               # VAD.C:126-129
        frm_zero = 0
        for h in range(159):                                                     # VAD.C:132-157
            if vc[i + h] >= a_thl:
                last_sig = 2
            elif vc[i + h] < b_thl:
                last_sig = 1
            w = vc[i + h + 1]
            if w >= a_thl:
                frm_zero += last_sig == 1
            elif w < b_thl:
                frm_zero += last_sig == 2
        zeros.append(frm_zero)
        i += 80
    return np.array(sums, np.int64), np.array(zeros, np.int64), np.array(entry, np.int64)


def vad_active(frames, atap):
    """VAD.C:164: a frame is active when frm_sum > s_thl or frm_zero > z_thl"""
    frm_sum, frm_zero = frames[0], frames[1]
    return (frm_sum > int(atap["s_thl"])) | (frm_zero > int(atap["z_thl"]))


def vad_fsm(active, cap=None):
    """the endpoint FSM of VAD.C:164-216 over a frame-activity sequence: [(start, end)], end = NULL for a segment still
    open when the frames run out; cap: the VAD returns once cap segments have closed (max_vc_con = 3, VAD.C:202-205)"""
    cur, front, back, segs = 0, 0, 0, []
    for k, a in enumerate(active):
        i = 80 * k
        if a:                                                                    # VAD.C:164-187
            if cur == 0:
                cur, front = 1, 1
            elif cur == 1:
                front += 1
                if front >= 8:
                    cur, front = 2, 0
                    segs.append([i - 7 * 80, NULL])
            elif cur == 3:
                back, cur = 0, 2
        else:                                                                    # VAD.C:188-216
            if cur == 2:
                cur, back = 3, 1
            elif cur == 3:
                back += 1
                if back >= 11:
                    cur, back = 0, 0
                    segs[-1][1] = i - 11 * 80 + 160
                    if cap is not None and len(segs) == cap:
                        break
            elif cur == 1:
                front, cur = 0, 0
    return [tuple(s) for s in segs]


def py_vad(vc, n, atap, cap=None):
    """VAD.C:97-218 on the first n samples: [(start, end)] (see vad_fsm)"""
    return vad_fsm(vad_active(vad_frames(vc, n, atap), atap), cap)


def seg_table(segs, cap=3):
    """a [cap, 2] u32 table of segment offsets as VAD writes them (NULL where no segment opened or closed)"""
    t = np.full((cap, 2), NULL, np.uint32)
    for j, s in enumerate(segs[:cap]):
        t[j] = s
    return t


def py_vad_long(vc, n, atap):
    """the long-form VAD (VAD.C:97-218 without max_vc_con): [(start, end)], end = NULL for a segment still open when the
    frames run out"""
    return py_vad(vc, n, atap)


# ---- the host's launch plan of the connected-word calls, restated ----------------------------------------------------
PIECE_CHUNK = 8192          # kPieceChunk, csrc/sr_api.cu
GRAM_REC_BYTES = 1 << 28    # kGramRecBytes, csrc/sr_api.cu
SEQ_CHUNK = 1 << 20         # kSeqChunk, csrc/sr_common.cuh


def pieces(F):
    """get_mfcc pieces of segments of F frames: ceil(F / 119)"""
    return (np.asarray(F, np.int64) + MAX_FRM - 1) // MAX_FRM


def piece_plan(counts):
    """pieces counts[r] of each row (capture order, then segment order) through launches of PIECE_CHUNK: (launches, the
    rows holding the last piece of a launch and the first of the next plus the first and last row with pieces, row
    slices [lo, hi) of at most PIECE_CHUNK pieces each)"""
    counts = np.asarray(counts, np.int64)
    owner = np.repeat(np.arange(len(counts)), counts)
    launches = -(-len(owner) // PIECE_CHUNK)
    edge = {int(owner[0]), int(owner[-1])}
    for k in range(1, launches):
        edge |= {int(owner[k * PIECE_CHUNK - 1]), int(owner[k * PIECE_CHUNK])}
    slices, lo, n = [], 0, 0
    for r, c in enumerate(counts):
        if n + c > PIECE_CHUNK:
            slices.append((lo, r))
            lo, n = r, 0
        n += int(c)
    slices.append((lo, len(counts)))
    return launches, edge, slices


def record_cuts(N, S):
    """run_grammar's launch boundaries [0, ..., B]: a cut before sequence b when rows && (rows + N[b]) * S * 8 > 2^28"""
    cuts, rows = [0], 0
    for b, n in enumerate(np.asarray(N, np.int64).tolist()):
        if rows and (rows + n) * S * 8 > GRAM_REC_BYTES:
            cuts.append(b)
            rows = 0
        rows += n
    return cuts + [len(N)]


def seq_launches(cuts):
    """the sequence ranges [lo, hi) of the kernel launches of a plan whose launch boundaries are cuts [0, ..., B] (K6:
    [0, B]; K6g: record_cuts), each cut range launched in chunks of SEQ_CHUNK"""
    return [(b0, min(b0 + SEQ_CHUNK, hi)) for lo, hi in zip(cuts[:-1], cuts[1:]) for b0 in range(lo, hi, SEQ_CHUNK)]


def launch_sample(edge, B, n, rng):
    """the indices in edge plus random ones, n in all (or all of edge when it is larger), sorted"""
    edge = sorted(set(int(e) for e in edge))
    rest = np.setdiff1d(np.arange(B), edge)
    pick = rng.choice(rest, min(max(n - len(edge), 0), len(rest)), replace=False)
    return np.array(sorted(edge + [int(p) for p in pick]), np.int64)
