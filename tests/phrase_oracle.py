"""CPU oracle of tantivy's phrase-query path, restated in Python independently of the CUDA library (test infrastructure).

  PositionSerializer / PositionReader           tantivy/src/positions/{serializer.rs,reader.rs}
  positions_with_offset                         tantivy/src/postings/segment_postings.rs:233-254
  intersection*, PhraseScorer                   tantivy/src/query/phrase_query/phrase_scorer.rs
  Bm25Weight::for_terms / score                 tantivy/src/query/bm25.rs:98-196
  for_each_pruning_scorer + TopNComputer        exact top-k by (score desc, doc asc)

An index here is a dict: fieldnorm_ids (u8 per doc) and, per term, `docs` (ascending) and `positions` (one ascending array
per posting).  All f32 arithmetic goes through numpy float32 scalars (IEEE round-to-nearest, no contraction)."""
import ctypes as C

import numpy as np

_libm = C.CDLL("libm.so.6")
_libm.logf.restype = C.c_float
_libm.logf.argtypes = [C.c_float]
F = np.float32


# ---- positions codec ---------------------------------------------------------------------------------------------------
def _vint(v):
    out = bytearray()
    while v >= 128:
        out.append(v & 127)
        v >>= 7
    out.append(v | 128)
    return out


def _bitpack4x(vals):
    """BitPacker4x::compress of 128 u32: width = bits of the largest value; value k goes to lane k % 4, slot k // 4, each
    lane a little-endian bit stream over 32-bit words, word w of lane l at u32 index 4w + l."""
    w = max(int(v) for v in vals).bit_length()
    words = [0] * (4 * w)
    for lane in range(4):
        acc = 0
        for slot in range(32):
            acc |= int(vals[slot * 4 + lane]) << (slot * w)
        for i in range(w):
            words[4 * i + lane] = (acc >> (32 * i)) & 0xFFFFFFFF
    return w, np.array(words, np.uint32).tobytes()


def serialize_positions(deltas):
    """PositionSerializer.write_positions_delta(deltas) + close_term(): the bytes of one term."""
    widths, body = bytearray(), bytearray()
    deltas = [int(x) for x in deltas]
    nfull = len(deltas) // 128
    for b in range(nfull):
        w, packed = _bitpack4x(deltas[b * 128:(b + 1) * 128])
        widths.append(w)
        body += packed
    for x in deltas[nfull * 128:]:
        body += _vint(x)
    return bytes(_vint(nfull) + widths + body)


def read_positions(data, offset, n):
    """PositionReader::open + read(offset, n): the deltas [offset, offset + n) of one term's bytes."""
    data = bytes(data)
    nblk, sh, p = 0, 0, 0
    while True:
        b = data[p]; p += 1
        nblk |= (b & 127) << sh
        if b & 128:
            break
        sh += 7
    widths = data[p:p + nblk]; p += nblk
    vals = []
    for w in widths:
        words = np.frombuffer(data[p:p + 16 * w], np.uint32).astype(object) if w else []
        p += 16 * w
        for k in range(128):
            if w == 0:
                vals.append(0)
                continue
            lane, slot = k % 4, k // 4
            acc = 0
            for i in range(w):
                acc |= int(words[4 * i + lane]) << (32 * i)
            vals.append((acc >> (slot * w)) & ((1 << w) - 1))
    v, sh = 0, 0
    for b in data[p:]:
        v |= (b & 127) << sh
        sh += 7
        if b & 128:
            vals.append(v); v, sh = 0, 0
    assert offset + n <= len(vals)
    return np.array(vals[offset:offset + n], np.uint32)


def positions_file(index):
    """The field's `.pos` file: every term's positions, deltas restarting at each posting.  Returns (bytes, off, len)."""
    blob, off, ln = bytearray(), [], []
    for t in index["terms"]:
        deltas = []
        for pos in t["positions"]:
            prev = 0
            for x in pos:
                deltas.append((int(x) - prev) & 0xFFFFFFFF)
                prev = int(x)
        b = serialize_positions(deltas)
        off.append(len(blob)); ln.append(len(b))
        blob += b
    return np.frombuffer(bytes(blob), np.uint8), np.array(off, np.uint64), np.array(ln, np.uint64)


# ---- intersections (phrase_scorer.rs:60-345) ---------------------------------------------------------------------------
def intersection_exists(left, right):
    i = j = 0
    while i < len(left) and j < len(right):
        if left[i] < right[j]:
            i += 1
        elif left[i] == right[j]:
            return True
        else:
            j += 1
    return False


def intersection_count(left, right):
    i = j = c = 0
    while i < len(left) and j < len(right):
        if left[i] < right[j]:
            i += 1
        elif left[i] == right[j]:
            c += 1; i += 1; j += 1
        else:
            j += 1
    return c


def intersection(left, right):
    """returns the new left"""
    out, i, j = [], 0, 0
    while i < len(left) and j < len(right):
        if left[i] < right[j]:
            i += 1
        elif left[i] == right[j]:
            out.append(left[i]); i += 1; j += 1
        else:
            j += 1
    return out


def intersection_count_with_slop(left, right, slop, update_left):
    """returns (count, new left or None)"""
    i = j = c = 0
    out = []
    while i < len(left) and j < len(right):
        lv, rv = left[i], right[j]
        if abs(lv - rv) <= slop:
            while i + 1 < len(left) and left[i + 1] <= rv:
                i += 1
            out.append(rv)
            c += 1; i += 1; j += 1
        elif lv < rv:
            i += 1
        else:
            j += 1
    return c, (out if update_left else None)


def intersection_exists_with_slop(left, right, slop):
    i = j = 0
    while i < len(left) and j < len(right):
        lv, rv = left[i], right[j]
        if abs(lv - rv) <= slop:
            return True
        if lv < rv:
            i += 1
        else:
            j += 1
    return False


def intersection_count_with_carrying_slop(left, left_slops, right, max_slop, update_left):
    """returns (count, new left, new left_slops); slops are u8 (`as u8` truncates), an empty left_slops means 0 so far.
    `slop_so_far as u32 + abs_diff` is a u32 add that wraps in the reference's release build (phrase_scorer.rs:270,297,317,
    327): a slop so far of s >= 1 and two positions at least 2^32 - s apart give a distance below s, which matches."""
    if not left or not right:
        return 0, ([] if update_left else left), ([] if update_left else left_slops)
    pb, sb = [], []

    def add(s, v):
        if not update_left:
            return
        if pb and pb[-1] == v:
            sb[-1] = min(sb[-1], s & 255)
        else:
            pb.append(v); sb.append(s & 255)

    i = j = count = 0
    while True:
        lv = left[i]
        sso = left_slops[i] if i < len(left_slops) else 0
        rv = right[j]
        dist = (sso + abs(lv - rv)) & 0xFFFFFFFF
        if dist <= max_slop:
            if lv < rv:
                smaller, larger, si, sp = lv, rv, i, left
            else:
                smaller, larger, si, sp = rv, lv, j, right
            new_slop = dist
            add(new_slop, smaller)
            while si + 1 < len(sp):
                nv = sp[si + 1]
                if nv > larger:
                    break
                si += 1
                new_slop = (sso + abs(nv - larger)) & 0xFFFFFFFF
                add(new_slop, nv)
            add(new_slop, larger)
            count += 1; i += 1; j += 1
        elif lv < rv:
            i += 1
        else:
            j += 1
        if i >= len(left) or j >= len(right):
            if i >= len(left):
                lv = left[-1]
                s0 = left_slops[-1] if left_slops else 0
                for r in right[j:]:
                    ns = (abs(lv - r) + s0) & 0xFFFFFFFF
                    if ns <= max_slop:
                        add(ns, r)
            else:
                rv = right[-1]
                for li in range(i, len(left)):
                    s0 = left_slops[li] if li < len(left_slops) else 0
                    ns = (abs(left[li] - rv) + s0) & 0xFFFFFFFF
                    if ns <= max_slop:
                        add(ns, left[li])
            break
    if update_left:
        return count, pb, sb
    return count, left, left_slops


# ---- PhraseScorer (phrase_scorer.rs:412-505) ---------------------------------------------------------------------------
def _match(lists, slop, scoring):
    """lists: the shifted positions of every docset in docset order.  Returns the phrase count (scoring) or 1/0 (exists)."""
    n = len(lists)
    left, left_slops = list(lists[0]), []
    right = None
    for i in range(1, n - 1):
        right = list(lists[i])
        if slop > 0:
            if n > 2:
                _, left, left_slops = intersection_count_with_carrying_slop(left, left_slops, right, slop, True)
            else:
                _, left = intersection_count_with_slop(left, right, slop, True)
        else:
            left = intersection(left, right)
        if not left:
            return 0
    right = list(lists[n - 1])
    if scoring:
        if slop > 0:
            if n > 2:
                return intersection_count_with_carrying_slop(left, left_slops, right, slop, False)[0]
            return intersection_count_with_slop(left, right, slop, False)[0]
        return intersection_count(left, right)
    if slop > 0:
        return 1 if intersection_exists_with_slop(left, right, slop) else 0
    return 1 if intersection_exists(left, right) else 0


def idf(doc_freq, doc_count):
    x = (F(doc_count - doc_freq) + F(0.5)) / (F(doc_freq) + F(0.5))
    return F(_libm.logf(float(F(1.0) + x)))


def tf_cache(avg_fieldnorm, fieldnorm_values):
    fn = np.asarray(fieldnorm_values, np.float32)
    return (F(1.2) * ((F(1.0) - F(0.75)) + (F(0.75) * fn) / F(avg_fieldnorm))).astype(np.float32)


def bm25_weight_for_terms(doc_freqs, total_num_docs):
    """Bm25Weight::for_terms(..).weight: idf of one term, or the f32 sum of the idfs in the order given, times (1 + K1)."""
    if len(doc_freqs) == 1:
        s = idf(doc_freqs[0], total_num_docs)
    else:
        s = F(0.0)
        for d in doc_freqs:
            s = F(s + idf(d, total_num_docs))
    return F(s * (F(1.0) + F(1.2)))


def phrase_search(index, terms, offsets=None, slop=0, scoring=True, weight=None, cache=None, k=None):
    """PhraseWeight::for_each_pruning + TopNComputer over one segment.  terms: term ids in offset order (None = a term the
    segment does not hold).  Returns [(score f32, doc)] in (score desc, doc asc) order, at most k."""
    offsets = list(range(len(terms))) if offsets is None else list(offsets)
    if any(t is None for t in terms):
        return []
    tl = index["terms"]
    max_off = max(offsets)
    docsets = [(t, max_off - o) for t, o in zip(terms, offsets)]
    docsets.sort(key=lambda p: len(tl[p[0]]["docs"]))   # Intersection::new: stable sort by size_hint
    common = None
    for t, _ in docsets:
        d = np.asarray(tl[t]["docs"], np.int64)
        common = d if common is None else np.intersect1d(common, d, assume_unique=True)
    hits = []
    for doc in common:
        lists = []
        for t, shift in docsets:
            i = int(np.searchsorted(tl[t]["docs"], doc))
            lists.append([(int(x) + shift) & 0xFFFFFFFF for x in tl[t]["positions"][i]])
        c = _match(lists, slop, scoring)
        if c == 0:
            continue
        if scoring:
            tf = F(c)
            s = F(weight * (tf / (tf + cache[index["fieldnorm_ids"][doc]])))
        else:
            s = F(1.0)
        hits.append((s, int(doc)))
    hits.sort(key=lambda h: (-float(h[0]), h[1]))
    return hits if k is None else hits[:k]


def build_index(texts):
    """Documents tokenized by lowercase whitespace split (what the reference tests' TEXT field gives these inputs).
    Returns (index, vocabulary {token: term id}); fieldnorm ids are the token counts (all < 24 here, where the code is
    the identity)."""
    vocab, postings = {}, {}
    lens = []
    for doc, text in enumerate(texts):
        toks = text.lower().split()
        lens.append(len(toks))
        for pos, tok in enumerate(toks):
            vocab.setdefault(tok, len(vocab))
            postings.setdefault(vocab[tok], {}).setdefault(doc, []).append(pos)
    assert max(lens) < 24
    terms = []
    for t in range(len(vocab)):
        ds = sorted(postings[t])
        terms.append({"docs": np.array(ds, np.uint32), "positions": [np.array(postings[t][d], np.uint32) for d in ds]})
    return {"fieldnorm_ids": np.array(lens, np.uint8), "terms": terms, "total_num_tokens": int(sum(lens))}, vocab
