"""Inputs, float64 references and a rounding model of the batched decode step's per-row kernels (batch.cu), shared by
tests/test_gpu_batch_kernels.py (one launch at a time through tests/batchcheck) and tests/test_batch_kernels_cpu.py (the bounds
rehearsed on the CPU, and evidence that they have teeth).

Attention bound: the one every fp16-P attention kernel of the project meets (kernel_ref.attention_check): |O - O_ref| <=
2^-9 max|V| per head and rel-L2 <= 1e-3.  The tensor-core kernel rounds q * scale and P to fp16 and writes fp16; a P below 2^-24
underflows to zero, which adds at most L 2^-25 max|V| (2.4e-4 max|V| at L = 8 192), so the batch-1 kernel's 1e-4 bound does not
apply here.  attn_model() restates the kernel's roundings in numpy so that the bound can be checked on every case without a GPU."""
import numpy as np

import kernel_ref as R

MAX_BATCH = 128
PAGE = R.KV_PAGE
NAN16 = np.uint16(0x7E5A)            # poison bits: a quiet NaN no kernel writes
SENT16 = np.uint16(0x7E5B)
ROPE_BASE = 500000.0

STEP_STATE = np.dtype([("pos", "<i4"), ("token", "<i4"), ("n_prompt", "<i4"), ("out_idx", "<i4"), ("done", "<i4"), ("ignore_eos", "<i4"),
                       ("n_stop", "<i4"), ("stop_ids", "<i4", (8,)), ("bar_base", "<u4"), ("temperature", "<f4"), ("top_k", "<i4"),
                       ("top_p", "<f4"), ("seed_lo", "<u4"), ("seed_hi", "<u4"), ("min_p", "<f4"), ("pen_last_n", "<i4"),
                       ("repeat_penalty", "<f4"), ("presence_penalty", "<f4"), ("frequency_penalty", "<f4"), ("json", "<i4")])
BATCH_CTL = np.dtype([("n_rows", "<i4"), ("row_slot", "<i4", (MAX_BATCH,))])
BATCH_OUT = np.dtype([("token", "<i4"), ("logprob", "<f4"), ("done", "<i4"), ("pos", "<i4")])
SAMPLE_PARTS, SAMPLE_THREADS = 8, 512          # batch_sample_greedy_kernel: CTAs per row, threads per CTA
SAMPLE_ROW_FLOATS = 3 * SAMPLE_PARTS + 1


def attn_splits_for(bucket, n_kv, n_sm):
    """engine_batch.cu: the split count the batched step launches with"""
    return max(1, min(16, (2 * n_sm) // max(1, n_kv * bucket)))


def rope_tables(n_pos, hd):
    from oracle import llama_oracle as O
    return O.rope_table(n_pos, hd, ROPE_BASE)


# ---- attention launch cases -------------------------------------------------------------------------------------------------
class AttnCase:
    """One batched attention launch: `positions[r]` is the position row r processes (its newest row); row r's sequence lives in
    slot `slots[r]`.  Physical pages are shuffled; one poison page (NaN) stands behind every table entry past a row's pages, and
    a few pages nobody owns are NaN too.  In each row's last page the slots past its position hold stale data (`stale`: finite
    random values, 'max' = +-65504, 'inf' = +-inf), as a page back from the pool does, and the newest slot holds a previous
    owner's finite row, which the launch must overwrite.  share = (a, b, k): row b's first k pages are row a's."""

    def __init__(self, hd, n_head, n_kv, S, positions, bucket=None, slots=None, share=None, stale="finite", seed=0):
        rng = np.random.Generator(np.random.PCG64(
            [seed, hd, n_head, n_kv, S, len(positions), int(sum(positions)), bucket or 0, ("finite", "max", "inf").index(stale)]))
        self.hd, self.n_head, self.n_kv, self.S, self.stale = hd, n_head, n_kv, S, stale
        self.pos = np.asarray(positions, np.int64)
        self.n_rows = len(positions)
        self.bucket = bucket or self.n_rows
        self.slots = np.asarray(slots if slots is not None else np.arange(self.n_rows), np.int64)
        self.scale = np.float32(1.0 / np.sqrt(hd))
        self.qd, self.kvd = n_head * hd, n_kv * hd
        self.ld = self.qd + 2 * self.kvd
        npg = self.pos // PAGE + 1
        self.n_pages = npg
        self.stride = int(npg.max()) + 2
        shared = {}                                     # (row, page) -> (row, page) whose physical page it uses
        if share is not None:
            a, b, k = share
            assert k * PAGE <= min(self.pos[a], self.pos[b]), "shared pages must lie below both rows' newest position"
            for j in range(k):
                shared[(b, j)] = (a, j)
        n_own = int(npg.sum()) - len(shared)
        n_phys = n_own + 4
        perm = rng.permutation(n_phys)
        self.poison = int(perm[0])
        nxt = 1
        self.tables = np.full((MAX_BATCH, self.stride), self.poison, np.int32)
        for r in range(self.n_rows):
            for j in range(npg[r]):
                if (r, j) in shared:
                    a, ja = shared[(r, j)]
                    self.tables[self.slots[r], j] = self.tables[self.slots[a], ja]
                else:
                    self.tables[self.slots[r], j] = perm[nxt]
                    nxt += 1
        self.n_phys = n_phys
        shape = (n_phys, n_kv, PAGE, hd)
        self.kc = np.full(shape, NAN16, np.uint16)
        self.vc = self.kc.copy()
        for r in range(self.n_rows):
            n = int(npg[r]) * PAGE
            k = rng.standard_normal((n, n_kv, hd)).astype(np.float16)
            v = rng.standard_normal((n, n_kv, hd)).astype(np.float16)
            p = int(self.pos[r])
            tail = slice(p + 1, n)
            if stale == "max":
                k[tail] = np.float16(65504.0) * rng.choice([-1, 1], size=k[tail].shape)
                v[tail] = np.float16(65504.0) * rng.choice([-1, 1], size=v[tail].shape)
            elif stale == "inf":
                k[tail] = np.float16(np.inf) * rng.choice([-1, 1], size=k[tail].shape)
                v[tail] = np.float16(np.inf) * rng.choice([-1, 1], size=v[tail].shape)
            for j in range(npg[r]):
                if (r, j) in shared:
                    continue
                ph = self.tables[self.slots[r], j]
                self.kc[ph] = k[j * PAGE:(j + 1) * PAGE].transpose(1, 0, 2).view(np.uint16)
                self.vc[ph] = v[j * PAGE:(j + 1) * PAGE].transpose(1, 0, 2).view(np.uint16)
        self.prev_k = np.stack([self.row_at(self.kc, r, int(self.pos[r])) for r in range(self.n_rows)])     # the previous owner's rows
        self.prev_v = np.stack([self.row_at(self.vc, r, int(self.pos[r])) for r in range(self.n_rows)])
        self.qkv = rng.standard_normal((self.bucket, self.ld)).astype(np.float32)
        self.cos, self.sin = rope_tables(int(self.pos.max()) + 2, hd)
        self.ctl = np.zeros(1, BATCH_CTL)
        self.ctl["n_rows"] = self.n_rows
        self.ctl["row_slot"][0, :self.n_rows] = self.slots
        self.st = np.zeros(MAX_BATCH, STEP_STATE)
        self.st["pos"][self.slots] = self.pos
        # what the launch appends: K rotated in float64 with the fp32 tables, V as numpy's float32 -> float16
        self.q_ref = R.rope_rows(self.qkv[:self.n_rows, :self.qd].astype(np.float64), self.pos, self.cos, self.sin, hd)
        self.k_raw = self.qkv[:self.n_rows, self.qd:self.qd + self.kvd].astype(np.float64)
        self.k_ref = R.rope_rows(self.k_raw, self.pos, self.cos, self.sin, hd)
        self.v16 = self.qkv[:self.n_rows, self.qd + self.kvd:].astype(np.float16)
        self.kc_after, self.vc_after = self.kc.copy(), self.vc.copy()
        self.newest = np.zeros(shape[:1] + shape[2:3], bool)         # [page][slot]: the rows the launch writes
        for r in range(self.n_rows):
            ph, t = self.slot_of(r)
            self.kc_after[ph, :, t] = self.k_ref[r].astype(np.float16).reshape(n_kv, hd).view(np.uint16)
            self.vc_after[ph, :, t] = self.v16[r].reshape(n_kv, hd).view(np.uint16)
            self.newest[ph, t] = True

    def slot_of(self, r, p=None):
        p = int(self.pos[r]) if p is None else p
        return int(self.tables[self.slots[r], p // PAGE]), p % PAGE

    def row_at(self, cache, r, p):
        ph, t = self.slot_of(r, p)
        return cache[ph, :, t].view(np.float16).astype(np.float64)

    def gather(self, cache, table_row, L, page_map=None):
        """logical rows [L, n_kv * hd] (float64) read through table_row; page_map: logical page -> logical page read instead"""
        lp = np.arange(L) // PAGE
        if page_map is not None:
            lp = page_map[lp]
        return cache[table_row[lp], :, np.arange(L) % PAGE].view(np.float16).astype(np.float64).reshape(L, -1)

    def kv(self, r, mutant=None):
        """the K / V rows row r attends over after the launch (float64 [pos + 1, n_kv * hd]), as a mutant sees them"""
        L = int(self.pos[r]) + 1
        table = self.tables[self.slots[r]]
        page_map = None
        if mutant == "neighbour_table":
            table = self.tables[self.slots[(r + 1) % self.n_rows]]
        elif mutant == "broken_reload":
            page_map = broken_reload_map(int(self.n_pages[r]), self.S)
        k = self.gather(self.kc_after, table, L, page_map)
        v = self.gather(self.vc_after, table, L, page_map)
        if mutant == "stale_newest":
            k[-1], v[-1] = self.prev_k[r].reshape(-1), self.prev_v[r].reshape(-1)
        elif mutant == "unrotated_k":
            k[-1] = self.k_raw[r].astype(np.float16)
        elif mutant in ("rot_pos-1", "rot_pos+1"):
            p = int(self.pos[r]) + (1 if mutant == "rot_pos+1" else -1)
            k[-1] = R.rope_rows(self.k_raw[r:r + 1], np.array([p]), self.cos, self.sin, self.hd)[0].astype(np.float16)
        return k, v

    def q(self, r, mutant=None):
        if mutant in ("rot_pos-1", "rot_pos+1"):
            p = int(self.pos[r]) + (1 if mutant == "rot_pos+1" else -1)
            return R.rope_rows(self.qkv[r:r + 1, :self.qd].astype(np.float64), np.array([p]), self.cos, self.sin, self.hd)[0]
        return self.q_ref[r]

    def kept_pages(self, r, mutant):
        """logical pages a page-dropping mutant still visits (None: every page)"""
        pg = np.arange(int(self.n_pages[r]))
        if mutant == "lost_warp":          # warp 1 of split 0 never ran: pages 0 + (1 + 4 j) S
            return pg[~((pg % self.S == 0) & ((pg // self.S) % 4 == 1))]
        if mutant == "drop_split1":
            return pg[pg % self.S != 1]
        return None

    def reference(self, r, mutant=None):
        """float64 softmax(q k^T scale) v of row r ([n_head * hd]) and the V rows the bound is taken over"""
        k, v = self.kv(r, mutant)
        q = self.q(r, mutant)
        keep = self.kept_pages(r, mutant)
        if keep is not None:
            rows = (keep[:, None] * PAGE + np.arange(PAGE)[None, :]).reshape(-1)
            rows = rows[rows < k.shape[0]]
            k, v = k[rows], v[rows]
        out = R.attention(q[None, :], k, v, k.shape[0] - 1, self.n_head, self.n_kv, self.hd, float(self.scale),
                          mutant="gqa_mod" if mutant == "gqa_mod" else None)
        return out[0], v

    def applies(self, r, mutant):
        """does `mutant` change row r's operation at all?"""
        p, npg, S = int(self.pos[r]), int(self.n_pages[r]), self.S
        if mutant == "lost_warp":
            return npg > S
        if mutant == "drop_split1":
            return S >= 2 and npg >= 2
        if mutant in ("unrotated_k", "rot_pos-1", "rot_pos+1"):
            return p >= 1
        if mutant == "broken_reload":
            return npg > 32 * 4 * S
        if mutant == "neighbour_table":
            return self.n_rows > 1
        if mutant == "gqa_mod":
            return self.n_kv > 1 and self.n_head > self.n_kv
        return True


def broken_reload_map(n_pages, S):
    """logical page read in place of each page when a warp's pages j >= 32 go through the cached entries of j - 32"""
    m = np.arange(n_pages)
    for pg in range(n_pages):
        s, c = pg % S, pg // S
        w, j = c % 4, c // 4
        if j >= 32:
            m[pg] = s + (w + 4 * (j % 32)) * S
    return m


def attn_distance(got, ref, v, n_head, n_kv, hd):
    """max(worst error / bound, rel-L2 / 1e-3): <= 1 passes"""
    if not np.isfinite(got).all():
        return np.inf
    ratio, rl2 = R.attention_check(got[None, :], ref[None, :], v, n_head, n_kv, hd)
    return max(ratio, rl2 / R.ATTN_REL_L2)


# ---- the kernel's roundings ---------------------------------------------------------------------------------------------
def _f32(x):
    return np.asarray(x, np.float64).astype(np.float32).astype(np.float64)


def _f16(x):
    return np.asarray(x, np.float64).astype(np.float16).astype(np.float64)


def attn_model(case, r):
    """batch_attn_mma_kernel's arithmetic for row r in numpy: q rotated in fp32, fp16(q * scale); per warp an online softmax page
    by page with P = exp(s - running max) rounded to fp16 for P V (l sums the unrounded fp32 P); the four warps merged, then the
    splits, in order; fp16 output.  The V rows of the last page past the position are zero (P = 0 there)."""
    hd, S, n_kv = case.hd, case.S, case.n_kv
    grp = case.n_head // n_kv
    L = int(case.pos[r]) + 1
    npg = int(case.n_pages[r])
    k, v = case.kv(r)
    q32 = _f32(case.q_ref[r])
    qh = _f16(_f32(q32 * np.float64(case.scale))).reshape(n_kv, grp, hd)
    J = -(-npg // (4 * S))                                     # pages per warp, rounded up
    tot = J * 4 * S
    kp = np.zeros((tot * PAGE, n_kv, hd))
    vp = np.zeros((tot * PAGE, n_kv, hd))
    kp[:L] = k.reshape(L, n_kv, hd)
    vp[:L] = v.reshape(L, n_kv, hd)
    s_all = _f32(np.einsum("kgd,lkd->kgl", qh, kp))            # [n_kv, grp, positions]
    s_all[..., L:] = -np.inf
    # page pg = (j * 4 + w) * S + s: view [n_kv, grp, J, 4, S, 16]
    s_all = s_all.reshape(n_kv, grp, J, 4, S, PAGE)
    vv = vp.reshape(J, 4, S, PAGE, n_kv, hd)
    valid = (np.arange(tot).reshape(J, 4, S) < npg)           # the page exists (a warp's loop covers only its own pages)
    m = np.full((n_kv, grp, 4, S), -np.inf)
    l = np.zeros((n_kv, grp, 4, S))
    o = np.zeros((n_kv, grp, 4, S, hd))
    with np.errstate(invalid="ignore", over="ignore"):
        for j in range(J):
            sv = s_all[:, :, j]                                  # [n_kv, grp, 4, S, 16]
            mx = sv.max(axis=-1)
            m_new = np.maximum(m, mx)
            corr = np.where(m == -np.inf, 0.0, _f32(np.exp(m - m_new)))
            p = _f32(np.exp(sv - m_new[..., None]))
            ps = _f32(p.sum(axis=-1))
            p16 = _f16(p)
            pv = np.einsum("kgwsp,wspkd->kgwsd", p16, vv[j])
            ok = valid[j][None, None]
            l = np.where(ok, _f32(l * corr + ps), l)
            o = np.where(ok[..., None], _f32(o * corr[..., None] + pv), o)
            m = np.where(ok, m_new, m)
    # the four warps of each split
    M = m.max(axis=2)                                           # [n_kv, grp, S]
    with np.errstate(invalid="ignore"):                        # a warp without pages: m = M = -inf, weight 0
        w = np.where(m == -np.inf, 0.0, _f32(np.exp(m - M[:, :, None, :])))
    den = _f32((w * l).sum(axis=2))
    acc = _f32((w[..., None] * o).sum(axis=2))                  # [n_kv, grp, S, hd]
    active = min(npg, S)
    if active == 1:
        out = acc[:, :, 0] / den[:, :, 0, None]
    else:
        M2 = M[:, :, :active].max(axis=2)
        w2 = _f32(np.exp(M[:, :, :active] - M2[..., None]))
        den2 = _f32((w2 * den[:, :, :active]).sum(axis=2))
        acc2 = _f32((w2[..., None] * acc[:, :, :active]).sum(axis=2))
        out = acc2 / den2[..., None]
    return _f16(out).reshape(-1)


# ---- the GPU cases (the CPU rehearsal runs on the same list) ---------------------------------------------------------------
ATTN_SHAPES = [(64, 4, 2), (128, 32, 8), (128, 64, 8), (128, 16, 8), (64, 16, 16)]      # (head_dim, n_head, n_kv)
ATTN_SPLITS = [1, 2, 3, 4, 7, 8, 16]


def engine_splits(n_kv):
    """the split counts the batched step picks for buckets 8 .. 128 on 114- and 132-SM parts: (bucket, S)"""
    out = {}
    for n_sm in (114, 132):
        for bucket in (8, 16, 32, 64, 128):
            out.setdefault(attn_splits_for(bucket, n_kv, n_sm), bucket)
    return sorted((b, s) for s, b in out.items())


def edge_positions(S):
    """positions at the page edges of a launch with S splits: the first pages, n_pages = S, 4 pages per warp round, fewer pages
    than splits"""
    p = {0, 15, 16, 17, 16 * S - 1, 16 * S, 16 * S + 1, 64 * S - 1, 64 * S, 64 * S + 1, 37}
    if S > 2:
        p.add(16 * (S // 2) - 1)
    return sorted(p)


def attn_cases():
    """(id, kwargs of AttnCase) of every GPU attention launch"""
    cases = []
    for hd, nh, nkv in ATTN_SHAPES:
        splits = sorted(set(ATTN_SPLITS) | {s for _b, s in engine_splits(nkv)})
        for S in splits:
            b = dict(engine_splits(nkv)).get(S)
            bucket = max(b or 0, len(edge_positions(S)))
            cases.append((f"hd{hd}-h{nh}-kv{nkv}-S{S}", dict(hd=hd, n_head=nh, n_kv=nkv, S=S, positions=edge_positions(S), bucket=bucket)))
    for S in (1, 2):        # a warp owns 64 / 128 pages at S = 1: the table reload runs 1 and 3 times
        cases.append((f"long-S{S}", dict(hd=128, n_head=32, n_kv=8, S=S, positions=[4095, 8191, 100])))
    for stale in ("max", "inf"):
        for hd, nh, nkv in ((64, 4, 2), (128, 32, 8)):
            cases.append((f"stale-{stale}-hd{hd}", dict(hd=hd, n_head=nh, n_kv=nkv, S=4, positions=[0, 5, 17, 40, 130, 301],
                                                        stale=stale)))
    cases.append(("layout", layout_kwargs()))
    return cases


def layout_kwargs():
    """bucket 128 with 100 rows, a permutation of slots up to 127, and rows 3 and 7 sharing their first two pages"""
    rng = np.random.Generator(np.random.PCG64(77))
    pos = rng.integers(0, 300, size=100)
    pos[3], pos[7] = 200, 140
    slots = rng.permutation(128)[:100]
    return dict(hd=128, n_head=32, n_kv=8, S=attn_splits_for(128, 8, 132), positions=pos.tolist(), bucket=128, slots=slots.tolist(),
                share=(3, 7, 2))


def private_copy_kwargs(kw):
    """the layout case with row 7's shared pages replaced by private pages holding the same bytes"""
    kw = dict(kw)
    kw["share"] = None
    return kw


ATTN_MUTANTS = ["lost_warp", "drop_split1", "stale_newest", "unrotated_k", "rot_pos-1", "rot_pos+1", "broken_reload",
                "neighbour_table", "gqa_mod"]


# ---- RoPE / KV append ----------------------------------------------------------------------------------------------------
def rope_bound(x_raw, hd):
    """2^-22 (|x0| + |x1|) per element of rows x_raw [rows, heads * hd] (the pair of each element)"""
    a = np.abs(x_raw).reshape(x_raw.shape[0], -1, 2).sum(axis=2)
    return 2.0 ** -22 * np.repeat(a, 2, axis=1)


def rope_mutant(x_raw, pos, cos, sin, hd, mutant):
    if mutant in ("pos-1", "pos+1"):
        return R.rope_rows(x_raw, np.maximum(pos + (1 if mutant == "pos+1" else -1), 0), cos, sin, hd)
    if mutant == "neox":      # pairs (x[i], x[i + hd / 2])
        rows = x_raw.shape[0]
        v = x_raw.reshape(rows, -1, hd)
        a, b = v[..., :hd // 2], v[..., hd // 2:]
        c = cos[pos].astype(np.float64)[:, None, :]
        s = sin[pos].astype(np.float64)[:, None, :]
        return np.concatenate([a * c - b * s, a * s + b * c], axis=-1).reshape(rows, -1)
    raise ValueError(mutant)


# ---- RMSNorm ---------------------------------------------------------------------------------------------------------------
def rmsnorm_rows(n, rows=5, seed=0):
    """rows of x: random, mean x^2 ~ 1e-6 (where eps matters), one 1e4 outlier, all zero, random at scale 30"""
    rng = np.random.Generator(np.random.PCG64([seed, n]))
    x = rng.standard_normal((rows, n)).astype(np.float32)
    x[1] *= np.float32(1e-3)
    x[2, n // 3] = np.float32(1e4)
    x[3] = 0.0
    x[4] *= np.float32(30.0)
    w = (1.0 + 0.5 * rng.standard_normal(n)).astype(np.float32)
    return x, w


def rmsnorm_ref(x, w, eps, mutant=None):
    """fp16(x w / sqrt(mean(x^2) + eps)) in float64 (before the fp16 rounding).  Mutants: 'no_eps', 'mean_n-1', 'w_shift'."""
    x = x.astype(np.float64)
    w = w.astype(np.float64)
    n = x.shape[1]
    ss = (x * x).sum(axis=1)
    ms = ss / (n - 1) if mutant == "mean_n-1" else ss / n
    e = 0.0 if mutant == "no_eps" else eps
    if mutant == "w_shift":
        w = np.roll(w, 1)
    with np.errstate(divide="ignore", invalid="ignore"):
        return x / np.sqrt(ms + e)[:, None] * w[None, :]


def rmsnorm_distance(got, ref):
    """worst |got - ref| in fp16 ulps of ref"""
    if not np.isfinite(got).all():
        return np.inf
    return float((np.abs(got - ref) / R.ulp16(ref)).max())


# ---- greedy draw ---------------------------------------------------------------------------------------------------------
def greedy_ref(logits):
    """(id, logprob) per row: the first maximum, -log sum exp(l - max) in float64"""
    l = logits.astype(np.float64)
    i = np.argmax(logits, axis=1)
    m = l[np.arange(l.shape[0]), i]
    with np.errstate(invalid="ignore"):
        s = np.where(np.isfinite(l), np.exp(l - m[:, None]), 0.0).sum(axis=1)
    return i, -np.log(s)


def greedy_lp_bound(n_vocab):
    """bound on |logprob - logprob_ref|.  The kernel sums s = sum exp(l - m) in fp32: each thread a run of at most
    ceil(n_vocab / 8 / 512) terms (each term and each rescale exp(m_old - m_new) within a few fp32 ulps, expf), then a 5-level
    shuffle tree, a 16-warp merge and an 8-part merge, each merge one rescale and one addition.  The relative error of s is at
    most (run + 5 + 15 + 7 + 4) 2^-23 to first order (every addition and every expf of at most 2 ulps); logf adds 2 ulps of the
    result and d(-log s) = ds / s.  So |d logprob| <= 2 (run + 31) 2^-23 + 2^-22 |logprob|: 2.4e-5 + 2.4e-7 |lp| at 151 936."""
    run = -(-n_vocab // SAMPLE_PARTS // SAMPLE_THREADS)
    return 2.0 * (run + 31) * 2.0 ** -23


def greedy_logits(n_vocab, rows, seed):
    """rows of logits with the edges the draw's tie rule and -inf handling must get right"""
    rng = np.random.Generator(np.random.PCG64([seed, n_vocab]))
    lg = (3.0 * rng.standard_normal((rows, n_vocab))).astype(np.float32)
    per = -(-n_vocab // SAMPLE_PARTS)
    # ties straddling a part boundary: per k - 1 and per k hold the maximum
    k = min(SAMPLE_PARTS - 1, max(1, (n_vocab - 1) // per))
    lg[0, per * k - 1] = lg[0, per * k] = 40.0
    # ties inside one part, across threads: the later index first in a thread's run, the earlier in another thread
    a = min(n_vocab - 1, 5 + SAMPLE_THREADS)
    lg[1, a] = lg[1, 5] = 40.0
    if rows > 2:       # all -inf but two entries, the winner in the last part
        lg[2] = -np.inf
        lg[2, n_vocab - 1] = 1.5
        lg[2, n_vocab // 3] = -2.0
    if rows > 3:       # all -inf but one
        lg[3] = -np.inf
        lg[3, n_vocab - 1] = -7.0
    if rows > 4:       # exact ties everywhere: every entry equal
        lg[4] = 0.25
    return lg


# ---- embedding gather --------------------------------------------------------------------------------------------------
def embed_bound(blocks, typ, n_vocab, cols):
    """per element: 2^-22 (|d sc q| + |dmin m|) for the quantised types (one or two fp32 roundings of each term), 0 for F16 / F32"""
    from oracle import gguf_synth as S, llama_oracle as O
    if typ in (S.F16, S.F32):
        return np.zeros((n_vocab, cols))
    if typ == S.Q4_K:
        b = np.ascontiguousarray(blocks).view(np.uint8).reshape(n_vocab, -1, 144)
        no_min, no_d = b.copy(), b.copy()
        no_min[:, :, 2:4] = 0
        no_d[:, :, 0:2] = 0
        a = np.abs(O.dequantize(no_min, typ, (n_vocab, cols))).astype(np.float64)
        c = np.abs(O.dequantize(no_d, typ, (n_vocab, cols))).astype(np.float64)
        return 2.0 ** -22 * (a + c)
    return 2.0 ** -22 * np.abs(O.dequantize(blocks, typ, (n_vocab, cols))).astype(np.float64)
