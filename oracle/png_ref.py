"""TEST INFRASTRUCTURE (oracle side): a numpy / pure-Python restatement of the PNG file `cv2.imencode('.png', img)`
writes with the libpng 1.6 and zlib 1.2.11 OpenCV 4.13 links, at OpenCV's PNG defaults (compression level 1, strategy
Z_RLE, filter SUB on every row, memLevel 8).

Stage by stage:
  - `filter_stream`: each row is a filter byte 1 (SUB) then the row's bytes minus the bytes one pixel to the left
    (mod 256); an image 1 pixel wide has filter byte 0 (NONE); BGR is stored as RGB; `[h][w]` is colour type 0,
    `[h][w][3]` colour type 2, 8 bits.
  - `tokens`: zlib's `deflate_rle` on that stream, in closed form.  A maximal run of R equal bytes is one literal,
    (R - 1) // 258 matches of length 258 (distance 1), then with r = (R - 1) % 258 one match of r if r >= 3, else r
    literals.  `deflate_rle_literal` is the loop itself (window, fill_window slides and row-by-row input as libpng
    feeds it) and proves the closed form, and the block cuts, on any input.
  - blocks: a block is flushed after every lit_bufsize - 1 = 16383 tokens (memLevel 8); the rest, possibly nothing,
    is the final block.
  - `flush_block`: trees.c's `build_tree` (heap ties broken by depth), `gen_bitlen` with its overflow repair,
    `gen_codes`, `build_bl_tree`, `scan_tree` / `send_tree`, and `_tr_flush_block`'s choice between a stored, a static
    and a dynamic block.  A stored block needs the block's bytes still in the window (`buf != NULL`); see `stored_ok`.
  - `zlib_stream`: the zlib header with libpng's window rule for streams of at most 16 KiB (`png_deflate_claim`
    lowers windowBits, zlib 1.2.11 raises 8 to 9, `optimize_cmf` rewrites CINFO in the first IDAT), the deflate
    bits, Adler-32.
  - `encode`: signature, IHDR, IDAT chunks of 8192 bytes of the zlib stream (the last one holds the rest), IEND.

Nothing in the package imports this module.
"""
import struct
import zlib

import numpy as np

MIN_MATCH, MAX_MATCH = 3, 258
LIT_BUFSIZE = 1 << (8 + 6)          # memLevel 8
BLOCK_TOKENS = LIT_BUFSIZE - 1      # _tr_tally flushes when last_lit == lit_bufsize - 1
MIN_LOOKAHEAD = MAX_MATCH + MIN_MATCH + 1
IDAT_BYTES = 8192                   # libpng's PNG_ZBUF_SIZE

L_CODES, D_CODES, BL_CODES, MAX_BITS, MAX_BL_BITS, END_BLOCK = 286, 30, 19, 15, 7, 256
HEAP_SIZE = 2 * L_CODES + 1
REP_3_6, REPZ_3_10, REPZ_11_138 = 16, 17, 18
EXTRA_LBITS = [0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0]
EXTRA_DBITS = [0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13]
EXTRA_BLBITS = [0] * 16 + [2, 3, 7]
BL_ORDER = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]


def _tables():
    """tr_static_init: length code and base of every match length - 3, and the static trees' lengths and codes"""
    length_code = [0] * 256
    base_length = [0] * 29
    length = 0
    for code in range(28):
        base_length[code] = length
        for _ in range(1 << EXTRA_LBITS[code]):
            length_code[length] = code
            length += 1
    length_code[length - 1] = 28     # length 258: code 285 without extra bits, not 284 + 5 bits
    slen = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
    bl_count = [0] * (MAX_BITS + 1)
    for v in slen:
        bl_count[v] += 1
    scode = _gen_codes(slen, 287, bl_count)
    dlen = [5] * D_CODES
    dcode = [_bi_reverse(n, 5) for n in range(D_CODES)]
    return length_code, base_length, slen, scode, dlen, dcode


def _bi_reverse(code, n):
    r = 0
    for _ in range(n):
        r = (r << 1) | (code & 1)
        code >>= 1
    return r


def _gen_codes(lens, max_code, bl_count):
    next_code = [0] * (MAX_BITS + 1)
    code = 0
    for bits in range(1, MAX_BITS + 1):
        code = (code + bl_count[bits - 1]) << 1
        next_code[bits] = code
    codes = [0] * len(lens)
    for n in range(max_code + 1):
        ln = lens[n]
        if ln:
            codes[n] = _bi_reverse(next_code[ln], ln)
            next_code[ln] += 1
    return codes


LENGTH_CODE, BASE_LENGTH, STATIC_LLEN, STATIC_LCODE, STATIC_DLEN, STATIC_DCODE = _tables()


# ---- filter -------------------------------------------------------------------------------------------------------

def check_image(img):
    """the images cv2.imencode('.png') takes here: u8, [h][w] or [h][w][3], no side 0"""
    a = np.asarray(img)
    if a.dtype != np.uint8 or a.ndim not in (2, 3) or (a.ndim == 3 and a.shape[2] != 3) or 0 in a.shape:
        raise ValueError("a PNG image must be u8 [h][w] or [h][w][3] with no side 0, got %s %s" % (a.dtype, a.shape))
    return a


def filter_type(width):
    """png_write_start_row drops SUB for an image 1 pixel wide, which leaves NONE (0); SUB (1) otherwise.  For such an
    image both give the same row bytes; only the filter byte differs."""
    return 0 if width == 1 else 1


def filter_stream(img):
    """the SUB-filtered stream libpng compresses: h rows of 1 + w * channels bytes"""
    a = check_image(img)
    if a.ndim == 3:
        a = a[:, :, ::-1]
    bpp = 1 if a.ndim == 2 else 3
    rows = np.ascontiguousarray(a).reshape(a.shape[0], -1)
    out = np.empty((rows.shape[0], rows.shape[1] + 1), np.uint8)
    out[:, 0] = filter_type(a.shape[1])
    out[:, 1:] = rows
    out[:, 1 + bpp:] -= rows[:, :-bpp]
    return out.ravel()


# ---- tokens -------------------------------------------------------------------------------------------------------
# A token is an int: 0..255 a literal, 256 + L a match of length L (always at distance 1).

def runs(s):
    """(start, length) of every maximal run of equal bytes"""
    s = np.asarray(s, np.uint8)
    starts = np.flatnonzero(np.r_[True, s[1:] != s[:-1]])
    return starts, np.diff(np.r_[starts, s.size])


def run_token_count(R):
    R = np.asarray(R, np.int64)
    q, r = (R - 1) // MAX_MATCH, (R - 1) % MAX_MATCH
    return 1 + q + np.where(r >= MIN_MATCH, 1, r)


def tokens(s):
    """deflate_rle's tokens in closed form (module docstring)"""
    s = np.asarray(s, np.uint8)
    st, R = runs(s)
    n = run_token_count(R)
    off = np.r_[0, np.cumsum(n)]
    T = int(off[-1])
    k = np.repeat(np.arange(st.size), n)
    i = np.arange(T) - off[k]
    q, r = (R[k] - 1) // MAX_MATCH, (R[k] - 1) % MAX_MATCH
    lit = s[st[k]].astype(np.int64)
    out = np.where(i == 0, lit,
                   np.where(i <= q, 256 + MAX_MATCH, np.where(r >= MIN_MATCH, 256 + r, lit)))
    return out


def token_bytes(t):
    t = np.asarray(t, np.int64)
    return np.where(t < 256, 1, t - 256)


def deflate_rle_literal(s, row_bytes, wbits=15):
    """zlib 1.2.11 `deflate_rle` run as libpng drives it: one deflate(Z_NO_FLUSH) per row of `row_bytes` bytes, then
    deflate(Z_FINISH) without input.  The window is followed by its absolute positions: `base` is the stream position
    of window[0], `end` that of the window's last byte read, and `fill_window` slides by w_size when strstart reaches
    w_size + MAX_DIST, as 1.2.11 does.  Returns (tokens, blocks) with one (first token, token count, block_start,
    stored_len, buf_ok, last) per flushed block; buf_ok is `block_start >= 0` in window terms."""
    s = np.asarray(s, np.uint8)
    N = s.size
    wsize = 1 << wbits
    max_dist = wsize - MIN_LOOKAHEAD
    st = dict(base=0, end=0, avail=0, fed=0, strstart=0, block_start=0, last_lit=0)
    toks, blocks = [], []

    def fill_window():
        while True:
            more = 2 * wsize - (st["end"] - st["base"])
            if st["strstart"] - st["base"] >= wsize + max_dist:
                st["base"] += wsize
                more += wsize
            if st["avail"] == 0:
                break
            n = min(st["avail"], more)
            st["end"] += n
            st["avail"] -= n
            if not (st["end"] - st["strstart"] < MIN_LOOKAHEAD and st["avail"] != 0):
                break

    def flush(last):
        bs = st["block_start"]
        blocks.append((len(toks) - st["last_lit"], st["last_lit"], bs, st["strstart"] - bs, bs - st["base"] >= 0,
                       last))
        st["block_start"] = st["strstart"]
        st["last_lit"] = 0

    def run(finish):
        while True:
            if st["end"] - st["strstart"] <= MAX_MATCH:
                fill_window()
                look = st["end"] - st["strstart"]
                if look <= MAX_MATCH and not finish:
                    return
                if look == 0:
                    break
            p = st["strstart"]
            look = st["end"] - p
            ml = 0
            if look >= MIN_MATCH and p > 0:
                prev = s[p - 1]
                if s[p] == prev and s[p + 1] == prev and s[p + 2] == prev:
                    seg = s[p:min(p + MAX_MATCH, st["end"])] != prev
                    ml = int(np.argmax(seg)) if seg.any() else seg.size
                    ml = min(ml, look)
            if ml >= MIN_MATCH:
                toks.append(256 + ml)
                st["strstart"] += ml
            else:
                toks.append(int(s[p]))
                st["strstart"] += 1
            st["last_lit"] += 1
            if st["last_lit"] == BLOCK_TOKENS:
                flush(False)
        flush(True)

    for r0 in range(0, N, row_bytes):
        st["avail"] += min(row_bytes, N - r0)
        run(False)
    run(True)
    return np.array(toks, np.int64), blocks


def stored_ok(stored_len):
    """`buf != NULL` of `_tr_flush_block` (the block's bytes are still in the window) as the closed form decides it.
    fill_window's j-th slide happens at a stream position >= 32768 j + 32506 (strstart >= w_size + MAX_DIST in window
    terms), so a block of at most 32506 bytes always starts inside the window.  A longer block may or may not,
    depending on where libpng's rows end, but such a block never takes the stored form: it holds at most 16383 tokens
    for more than 32506 bytes, and its static encoding (<= 9 bits a literal, <= 12 bits a 3-byte match, <= 18 bits
    any match) is shorter than its bytes.  `deflate_rle_literal` gives the exact flag, and the tests check that both
    make the same file."""
    return stored_len <= 32506


# ---- trees (trees.c) ----------------------------------------------------------------------------------------------

class _Tree:
    def __init__(self, elems, static_len, extra, base, max_length):
        self.elems, self.stree, self.extra, self.base, self.max_length = elems, static_len, extra, base, max_length
        size = 2 * elems + 1
        self.freq = [0] * size
        self.len = [0] * size     # dl.len
        self.dad = [0] * size     # dl.dad (the same field as len in C; each is read before the other is written)
        self.code = [0] * size
        self.max_code = -1


class _Block:
    def __init__(self):
        self.opt_len = 0
        self.static_len = 0
        self.bl_count = [0] * (MAX_BITS + 1)
        self.heap = [0] * HEAP_SIZE
        self.depth = [0] * HEAP_SIZE

    def _smaller(self, t, n, m):
        return t.freq[n] < t.freq[m] or (t.freq[n] == t.freq[m] and self.depth[n] <= self.depth[m])

    def _pqdownheap(self, t, k):
        heap = self.heap
        v = heap[k]
        j = k << 1
        while j <= self.heap_len:
            if j < self.heap_len and self._smaller(t, heap[j + 1], heap[j]):
                j += 1
            if self._smaller(t, v, heap[j]):
                break
            heap[k] = heap[j]
            k = j
            j <<= 1
        heap[k] = v

    def build_tree(self, t):
        heap, depth = self.heap, self.depth
        self.heap_len, self.heap_max = 0, HEAP_SIZE
        max_code = -1
        for n in range(t.elems):
            if t.freq[n] != 0:
                self.heap_len += 1
                heap[self.heap_len] = max_code = n
                depth[n] = 0
            else:
                t.len[n] = 0
        while self.heap_len < 2:
            if max_code < 2:
                max_code += 1
                node = max_code
            else:
                node = 0
            self.heap_len += 1
            heap[self.heap_len] = node
            t.freq[node] = 1
            depth[node] = 0
            self.opt_len -= 1
            if t.stree:
                self.static_len -= t.stree[node]
        t.max_code = max_code
        for n in range(self.heap_len // 2, 0, -1):
            self._pqdownheap(t, n)
        node = t.elems
        while True:
            n = heap[1]
            heap[1] = heap[self.heap_len]
            self.heap_len -= 1
            self._pqdownheap(t, 1)
            m = heap[1]
            self.heap_max -= 1
            heap[self.heap_max] = n
            self.heap_max -= 1
            heap[self.heap_max] = m
            t.freq[node] = t.freq[n] + t.freq[m]
            depth[node] = max(depth[n], depth[m]) + 1
            t.dad[n] = t.dad[m] = node
            heap[1] = node
            node += 1
            self._pqdownheap(t, 1)
            if self.heap_len < 2:
                break
        self.heap_max -= 1
        heap[self.heap_max] = heap[1]
        self._gen_bitlen(t)
        codes = _gen_codes(t.len, max_code, self.bl_count)
        for n in range(max_code + 1):
            t.code[n] = codes[n]

    def _gen_bitlen(self, t):
        heap = self.heap
        bl_count = self.bl_count
        for b in range(MAX_BITS + 1):
            bl_count[b] = 0
        t.len[heap[self.heap_max]] = 0
        overflow = 0
        h = self.heap_max + 1
        while h < HEAP_SIZE:
            n = heap[h]
            bits = t.len[t.dad[n]] + 1
            if bits > t.max_length:
                bits = t.max_length
                overflow += 1
            t.len[n] = bits
            h += 1
            if n > t.max_code:
                continue
            bl_count[bits] += 1
            xbits = t.extra[n - t.base] if n >= t.base else 0
            f = t.freq[n]
            self.opt_len += f * (bits + xbits)
            if t.stree:
                self.static_len += f * (t.stree[n] + xbits)
        if overflow == 0:
            return
        while True:
            bits = t.max_length - 1
            while bl_count[bits] == 0:
                bits -= 1
            bl_count[bits] -= 1
            bl_count[bits + 1] += 2
            bl_count[t.max_length] -= 1
            overflow -= 2
            if overflow <= 0:
                break
        h = HEAP_SIZE
        for bits in range(t.max_length, 0, -1):
            n = bl_count[bits]
            while n != 0:
                h -= 1
                m = heap[h]
                if m > t.max_code:
                    continue
                if t.len[m] != bits:
                    self.opt_len += (bits - t.len[m]) * t.freq[m]
                    t.len[m] = bits
                n -= 1

    @staticmethod
    def _scan_or_send(t, max_code, visit):
        """the run-length walk shared by scan_tree and send_tree; visit(kind, curlen, count) per emitted group"""
        prevlen, nextlen, count = -1, t.len[0], 0
        max_count, min_count = (138, 3) if nextlen == 0 else (7, 4)
        t.len[max_code + 1] = 0xFFFF    # guard
        for n in range(max_code + 1):
            curlen, nextlen = nextlen, t.len[n + 1]
            count += 1
            if count < max_count and curlen == nextlen:
                continue
            elif count < min_count:
                visit("lens", curlen, count)
            elif curlen != 0:
                visit("rep", curlen, count if curlen == prevlen else -count)
            elif count <= 10:
                visit("z10", 0, count)
            else:
                visit("z138", 0, count)
            count, prevlen = 0, curlen
            if nextlen == 0:
                max_count, min_count = 138, 3
            elif curlen == nextlen:
                max_count, min_count = 6, 3
            else:
                max_count, min_count = 7, 4

    def build_bl_tree(self, lt, dt, bt):
        def scan(kind, cur, count):
            if kind == "lens":
                bt.freq[cur] += count
            elif kind == "rep":
                if count < 0:
                    bt.freq[cur] += 1
                bt.freq[REP_3_6] += 1
            elif kind == "z10":
                bt.freq[REPZ_3_10] += 1
            else:
                bt.freq[REPZ_11_138] += 1
        self._scan_or_send(lt, lt.max_code, scan)
        self._scan_or_send(dt, dt.max_code, scan)
        self.build_tree(bt)
        max_blindex = BL_CODES - 1
        while max_blindex >= 3:
            if bt.len[BL_ORDER[max_blindex]] != 0:
                break
            max_blindex -= 1
        self.opt_len += 3 * (max_blindex + 1) + 5 + 5 + 4
        return max_blindex


class BitWriter:
    """deflate's LSB-first bit order; `bits` grows a Python int"""

    def __init__(self):
        self.acc, self.n = 0, 0

    def put(self, v, nbits):
        self.acc |= int(v) << self.n
        self.n += nbits

    def put_many(self, vals, lens):
        """many codes at once (numpy arrays of values and lengths)"""
        lens = np.asarray(lens, np.int64)
        if lens.size == 0:
            return
        off = np.r_[0, np.cumsum(lens)]
        total = int(off[-1])
        bit_idx = np.arange(total) - np.repeat(off[:-1], lens)
        bits = (np.repeat(np.asarray(vals, np.uint64), lens) >> bit_idx.astype(np.uint64)) & np.uint64(1)
        packed = np.packbits(bits.astype(np.uint8), bitorder="little")
        self.put(int.from_bytes(packed.tobytes(), "little"), total)

    def align(self):
        self.n = (self.n + 7) & ~7

    def tobytes(self):
        return self.acc.to_bytes((self.n + 7) // 8, "little")


def _token_codes(t, lcode, llen, dcode, dlen):
    """(value, length) of every token: the literal / length code, its extra bits and the distance code, packed"""
    t = np.asarray(t, np.int64)
    lcode, llen = np.asarray(lcode, np.int64), np.asarray(llen, np.int64)
    is_m = t >= 256
    lc = np.where(is_m, t - 256 - MIN_MATCH, 0)
    code = np.asarray(LENGTH_CODE, np.int64)[lc]
    sym = np.where(is_m, code + 257, t)
    v, n = lcode[sym], llen[sym]
    xb = np.where(is_m, np.asarray(EXTRA_LBITS, np.int64)[code], 0)
    xv = np.where(xb > 0, lc - np.asarray(BASE_LENGTH, np.int64)[code], 0)   # length 258: code 285, no extra bits
    v = v | np.where(is_m, xv << n, 0)
    n = n + xb
    v = v | np.where(is_m, dcode[0] << n, 0)
    n = n + np.where(is_m, dlen[0], 0)
    return v, n


def flush_block(bw, s, blk_tokens, block_start, stored_len, buf_ok, last):
    """_tr_flush_block at level 1: the block's trees, its form, and its bits into `bw`.  Returns the form
    (0 stored, 1 static, 2 dynamic)."""
    t = np.asarray(blk_tokens, np.int64)
    b = _Block()
    lt = _Tree(L_CODES, STATIC_LLEN, EXTRA_LBITS, 257, MAX_BITS)
    dt = _Tree(D_CODES, STATIC_DLEN, EXTRA_DBITS, 0, MAX_BITS)
    bt = _Tree(BL_CODES, None, EXTRA_BLBITS, 0, MAX_BL_BITS)
    is_m = t >= 256
    sym = np.where(is_m, np.asarray(LENGTH_CODE, np.int64)[np.where(is_m, t - 256 - MIN_MATCH, 0)] + 257, t)
    lt.freq[:L_CODES] = np.bincount(sym, minlength=L_CODES).tolist()
    lt.freq[END_BLOCK] = 1
    dt.freq[0] = int(is_m.sum())
    b.build_tree(lt)
    b.build_tree(dt)
    max_blindex = b.build_bl_tree(lt, dt, bt)
    opt_lenb = (b.opt_len + 3 + 7) >> 3
    static_lenb = (b.static_len + 3 + 7) >> 3
    if static_lenb <= opt_lenb:
        opt_lenb = static_lenb
    if stored_len + 4 <= opt_lenb and buf_ok:
        assert stored_len <= 0xFFFF
        bw.put(0 + int(last), 3)
        bw.align()
        bw.put(stored_len, 16)
        bw.put(~stored_len & 0xFFFF, 16)
        bw.put(int.from_bytes(np.asarray(s[block_start:block_start + stored_len]).tobytes(), "little"),
               8 * stored_len)
        form = 0
    elif static_lenb == opt_lenb:
        bw.put((1 << 1) + int(last), 3)
        v, n = _token_codes(t, STATIC_LCODE, STATIC_LLEN, STATIC_DCODE, STATIC_DLEN)
        bw.put_many(v, n)
        bw.put(STATIC_LCODE[END_BLOCK], STATIC_LLEN[END_BLOCK])
        form = 1
    else:
        bw.put((2 << 1) + int(last), 3)
        lcodes, dcodes, blcodes = lt.max_code + 1, dt.max_code + 1, max_blindex + 1
        bw.put(lcodes - 257, 5)
        bw.put(dcodes - 1, 5)
        bw.put(blcodes - 4, 4)
        for rank in range(blcodes):
            bw.put(bt.len[BL_ORDER[rank]], 3)

        def send(kind, cur, count):
            if kind == "lens":
                for _ in range(count):
                    bw.put(bt.code[cur], bt.len[cur])
            elif kind == "rep":
                if count < 0:      # curlen != prevlen: the length itself first
                    count = -count
                    bw.put(bt.code[cur], bt.len[cur])
                    count -= 1
                bw.put(bt.code[REP_3_6], bt.len[REP_3_6])
                bw.put(count - 3, 2)
            elif kind == "z10":
                bw.put(bt.code[REPZ_3_10], bt.len[REPZ_3_10])
                bw.put(count - 3, 3)
            else:
                bw.put(bt.code[REPZ_11_138], bt.len[REPZ_11_138])
                bw.put(count - 11, 7)
        _Block._scan_or_send(lt, lcodes - 1, send)
        _Block._scan_or_send(dt, dcodes - 1, send)
        v, n = _token_codes(t, lt.code[:L_CODES], lt.len[:L_CODES], dt.code[:D_CODES], dt.len[:D_CODES])
        bw.put_many(v, n)
        bw.put(lt.code[END_BLOCK], lt.len[END_BLOCK])
        form = 2
    if last:
        bw.align()
    return form


def deflate(s, tok=None, blocks=None):
    """the raw deflate stream of `s`.  Without `blocks`, the closed-form tokens cut every 16383 tokens with
    `stored_ok`; with the (tokens, blocks) of `deflate_rle_literal`, its blocks and buf flags.  Returns
    (bytes, forms)."""
    s = np.asarray(s, np.uint8)
    if blocks is None:
        tok = tokens(s)
        pos = np.r_[0, np.cumsum(token_bytes(tok))]
        T = tok.size
        blocks = []
        for b0 in range(0, T + 1, BLOCK_TOKENS):
            n = min(BLOCK_TOKENS, T - b0)
            last = b0 + BLOCK_TOKENS > T
            start, end = int(pos[b0]), int(pos[b0 + n])
            blocks.append((b0, n, start, end - start, stored_ok(end - start), last))
            if last:
                break
    bw = BitWriter()
    forms = [flush_block(bw, s, tok[b0:b0 + n], start, ln, ok, last) for b0, n, start, ln, ok, last in blocks]
    return bw.tobytes(), forms


def window_bits(data_size):
    """(windowBits given to deflateInit2, CINFO after optimize_cmf) for a filtered stream of `data_size` bytes"""
    wbits = 15
    if data_size <= 16384:
        half = 1 << (wbits - 1)
        while data_size + 262 <= half:
            half >>= 1
            wbits -= 1
    if wbits == 8:
        wbits = 9        # zlib 1.2.11 deflateInit2
    cinfo = wbits - 8
    if data_size <= 16384:
        half = 1 << (cinfo + 7)
        if data_size <= half:
            while True:
                half >>= 1
                cinfo -= 1
                if not (cinfo > 0 and data_size <= half):
                    break
    return wbits, cinfo


def zlib_header(data_size):
    """deflate's 2-byte header at level 1 (FLEVEL 0), with libpng's optimize_cmf CINFO"""
    _, cinfo = window_bits(data_size)
    cmf = 0x08 | (cinfo << 4)
    flg = 31 - ((cmf << 8) % 31)
    return bytes([cmf, flg])


def adler32(s):
    """Adler-32 (RFC 1950) by numpy partial sums: A = 1 + sum b, B = n + sum (n - i) b_i"""
    b = np.asarray(s, np.uint8).astype(np.int64)
    n = b.size
    A = (1 + int(b.sum())) % 65521
    B = (n + int(((n - np.arange(n)) * b).sum() % 65521)) % 65521
    return (B << 16) | A


def zlib_stream(s, literal=False, row_bytes=None):
    s = np.asarray(s, np.uint8)
    if literal:
        tok, blocks = deflate_rle_literal(s, row_bytes, window_bits(s.size)[0])
        body, _ = deflate(s, tok, blocks)
    else:
        body, _ = deflate(s)
    return zlib_header(s.size) + body + struct.pack(">I", adler32(s))


def _chunk(kind, data):
    return struct.pack(">I", len(data)) + kind + data + struct.pack(">I", zlib.crc32(kind + data) & 0xFFFFFFFF)


def encode(img, literal=False):
    """the bytes of cv2.imencode('.png', img)[1] (module docstring).  literal=True runs the deflate_rle loop."""
    a = check_image(img)
    h, w = a.shape[:2]
    s = filter_stream(a)
    z = zlib_stream(s, literal, s.size // h)
    ihdr = struct.pack(">IIBBBBB", w, h, 8, 0 if a.ndim == 2 else 2, 0, 0, 0)
    out = [b"\x89PNG\r\n\x1a\n", _chunk(b"IHDR", ihdr)]
    for o in range(0, len(z), IDAT_BYTES):
        out.append(_chunk(b"IDAT", z[o:o + IDAT_BYTES]))
    out.append(_chunk(b"IEND", b""))
    return np.frombuffer(b"".join(out), np.uint8)
