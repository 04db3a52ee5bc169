"""Where the two framing engines cut their input, restated on the host, and seeded inputs that put bytes on those cuts.

The produce kernel (csrc/sse_kernel.cu) stages one segment at a time through an 8 KiB window per warp; the tile kernel
(csrc/sse_fused.cu) packs segments into 48 KiB tiles, or walks a larger segment window by window. The constants are read from
the sources, so that a changed constant fails a CPU test instead of silently moving the seams away from the inputs; the
restatements say where each window, round and tile falls, and the GPU tests assert with them that an input sits on the seam it
is labelled with."""
from __future__ import annotations

import os
import re
from dataclasses import dataclass, field

import numpy as np

CSRC = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "inference_gateway_b200", "csrc")


def _constants() -> dict:
    out = {}
    for fn, names in (("sse_common.cuh", ("BUF", "LT_MAX", "DONE_MAX")),
                      ("sse_fused.cu", ("TILE", "MAX_TSEGS", "PLAN_GROUP", "JQ_CAP", "W_STOPS", "W_STRUCT", "REC_MAX", "NREC",
                                        "TS_WORDS", "F_THREADS"))):
        src = open(os.path.join(CSRC, fn)).read()
        for n in names:
            m = re.search(r"\b" + n + r"\s*=\s*(\d+)", src)
            assert m, f"{n} not found in {fn}"
            out[n] = int(m.group(1))
        if fn == "sse_fused.cu":
            m = re.search(r"\bLCAP\s*=\s*(\w+)\s*;", src)
            out["LCAP"] = out[m.group(1)] if m.group(1) in out else int(m.group(1))
    return out


K = _constants()
BUF, LT_MAX, DONE_MAX = K["BUF"], K["LT_MAX"], K["DONE_MAX"]
TILE, MAX_TSEGS, LCAP, PLAN_GROUP, JQ_CAP = K["TILE"], K["MAX_TSEGS"], K["LCAP"], K["PLAN_GROUP"], K["JQ_CAP"]
W_STOPS, W_STRUCT, REC_MAX, NREC, TS_WORDS = K["W_STOPS"], K["W_STRUCT"], K["REC_MAX"], K["NREC"], K["TS_WORDS"]


def r16(n: int) -> int:
    return (n + 15) & ~15


# ------------------------------------------------------------------ restatements
def plan_tiles(carry_lens, in_lens, live) -> list:
    """sse_plan_kernel: (first segment, segment count) of every tile, in segment order. A segment's region is its carry and its
    bytes, each padded to 16, or 0 for a finished or dead connection (which still counts toward MAX_TSEGS). Greedy within
    independent groups of PLAN_GROUP segments: a tile closes when the next region does not fit TILE or at MAX_TSEGS segments;
    a region larger than TILE gets a tile of its own (big_segment)."""
    n = len(in_lens)
    tiles = []
    for g0 in range(0, n, PLAN_GROUP):
        first, acc, cnt = g0, 0, 0
        i = g0
        while i < min(g0 + PLAN_GROUP, n):
            size = r16(int(carry_lens[i])) + r16(int(in_lens[i])) if live[i] else 0
            if acc + size <= TILE and cnt + 1 <= MAX_TSEGS:
                acc += size
                cnt += 1
                i += 1
            elif cnt == 0:
                tiles.append((i, 1))
                i += 1
                first = i
            else:
                tiles.append((first, cnt))
                first, acc, cnt = i, 0, 0
        if cnt:
            tiles.append((first, cnt))
    return tiles


def _newlines(stream: bytes, lo: int, hi: int) -> list:
    a = np.frombuffer(stream, dtype=np.uint8, count=hi - lo, offset=lo) if hi > lo else np.zeros(0, np.uint8)
    return (np.flatnonzero(a == 10) + lo).tolist()


@dataclass
class Window:
    s0: int                 # stream position of the window's first data byte (the stream is carry + body)
    s1: int                 # stream position one past its last byte
    base: int               # window offset of s0 (produce: the carried front is right-aligned to 16; tile: front or carry pad)
    lines: list = field(default_factory=list)     # stream positions of the '\n' of every line the window completes
    round_size: int = 0
    carried: int | None = None   # the last window: stream position of the tail held back (== s1: none; None: in the carry slot)
    to_long: bool = False        # produce: the tail continues in the carry slot (a whole window without '\n')
    long_end: int | None = None  # produce: the '\n' that completes a line assembled in the carry slot
    restart: int | None = None   # tile: stream position of the line the next window starts at
    no_newline: bool = False     # tile: a window after the first without '\n' (the connection fails)

    def offset(self, p: int) -> int:
        return p - self.s0 + self.base

    def rounds(self) -> list:
        """Lines per round, in order."""
        n = len(self.lines)
        return [min(self.round_size, n - i) for i in range(0, n, self.round_size)] if n else []


def produce_windows(carry: bytes, body: bytes, in_long: bool = False) -> list:
    """The produce kernel's windows over one segment (sse_stream_kernel, sse_kernel.cu:123-431): the carried tail is staged so
    that it ends at A = round16(pend), the window takes room = BUF - A more bytes, rounds hold at most LT_MAX lines, and a
    tail of BUF - 32 bytes or more, with bytes still to come, continues in the carry slot (in_long) until its '\n'."""
    stream = carry + body
    n = len(body)
    pend = 0 if in_long else len(carry)
    consumed = 0
    wins = []
    while True:
        A = r16(pend)
        nload = min(n - consumed, BUF - A)
        s0 = len(carry) + consumed - pend
        consumed += nload
        s1 = len(carry) + consumed
        w = Window(s0, s1, A - pend, round_size=LT_MAX)
        wins.append(w)
        pos = s0
        if in_long:
            nl = _newlines(stream, s0, s1)
            if not nl:
                w.to_long = True
                pend = 0
                if consumed >= n:
                    break
                continue
            w.long_end = nl[0]
            in_long = False
            pos = nl[0] + 1
        w.lines = _newlines(stream, pos, s1)
        if w.lines:
            pos = w.lines[-1] + 1
        tail = s1 - pos
        if consumed >= n:
            w.carried = pos
            break
        if tail >= BUF - 32:
            w.to_long = in_long = True
            pend = 0
            continue
        pend = tail
    return wins


def tile_windows(carry: bytes, body: bytes) -> list:
    """The tile kernel's windows over one segment alone in its tile: one window when its region fits TILE, else big_segment
    (sse_fused.cu:1658-1710): the first window holds the carry (right-aligned to 16) and TILE - round16(carry) input bytes;
    every later one restarts at the line the previous one left unterminated, from the 16-byte boundary below it (the front
    bytes before the line are blanked). Rounds hold at most LCAP lines. A later window without '\n' fails the connection."""
    stream = carry + body
    c, n = len(carry), len(body)
    if r16(c) + r16(n) <= TILE:
        w = Window(0, c + n, r16(c) - c, round_size=LCAP)
        w.lines = _newlines(stream, 0, c + n)
        w.carried = w.lines[-1] + 1 if w.lines else 0
        return [w]
    wins = []
    src, cl, front = 0, c, 0
    while True:
        Aw = r16(cl)
        nbytes = min(n - src, TILE - Aw)
        d0 = 0 if cl else c + src + front
        e = c + src + nbytes
        w = Window(d0, e, (Aw - cl) if cl else front, round_size=LCAP)
        wins.append(w)
        w.lines = _newlines(stream, d0, e)
        ts = w.lines[-1] + 1 if w.lines else d0
        if src + nbytes >= n:
            w.carried = ts
            break
        if ts == d0:
            w.no_newline = True
            break
        w.restart = ts
        X = ts - c
        src, front, cl = X & ~15, X & 15, 0
    return wins


def count_stops(payload: bytes) -> int:
    """Stop bytes of a payload (the tile kernel's stop bitmap, stage 1a): '"', '\\\\', '[', bytes below 0x20 and from 0x80."""
    a = np.frombuffer(payload, dtype=np.uint8)
    return int(np.count_nonzero((a == 0x22) | (a == 0x5C) | (a == 0x5B) | (a < 0x20) | (a >= 0x80)))


def count_structural(payload: bytes) -> int:
    """Structural stops of a payload (warp_replay): quotes that are not escaped, and '[' outside strings."""
    n, inside, i = 0, False, 0
    while i < len(payload):
        ch = payload[i]
        if inside and ch == 0x5C:
            i += 2
            continue
        if ch == 0x22:
            inside = not inside
            n += 1
        elif ch == 0x5B and not inside:
            n += 1
        i += 1
    return n


# ------------------------------------------------------------------ stream pieces
def chunk(content: bytes = b"x", fin: bytes = b"null", eol: bytes = b"\n\n") -> bytes:
    return b'data: {"choices":[{"index":0,"delta":{"content":"' + content + b'"},"finish_reason":' + fin + b"}]}" + eol


MIN_DATA = len(chunk(b"", eol=b"\n"))
USAGE = b'data: {"choices":[],"usage":{"prompt_tokens":3,"completion_tokens":5,"total_tokens":8}}\n\n'
END = chunk(b"bye", b'"stop"') + USAGE + b"data: [DONE]\n\n"
SHORT = b'data: {"choices":[]}\n'                                   # a decoded line of 21 bytes
STOP_LINE = b'data: {"choices":[{"delta":{},"finish_reason":"stop"}]}\n'
FIRST = chunk(b"first")


def data_line(n: int, eol: bytes = b"\n", fin: bytes = b"null", fill: bytes = b"abcdefgh ") -> bytes:
    """A content chunk of exactly n bytes, eol included."""
    k = n - len(chunk(b"", fin, eol))
    assert k >= 0, n
    return chunk((fill * (k // len(fill) + 1))[:k], fin, eol)


def filler(k: int) -> bytes:
    """Exactly k bytes of complete lines: content chunks of about 1,000 bytes, a comment line or a blank line for the rest."""
    out = []
    while k > 1000 + MIN_DATA:
        out.append(data_line(1000))
        k -= 1000
    if k >= MIN_DATA:
        out.append(data_line(k))
    elif k >= 2:
        out.append(b":" + b"p" * (k - 2) + b"\n")
    elif k == 1:
        out.append(b"\n")
    return b"".join(out)


@dataclass
class Case:
    """One connection's stream. cuts: explicit batch boundaries (a batch boundary is a seam too); meta: where the seam is."""
    label: str
    body: bytes
    cuts: tuple = ()
    meta: dict = field(default_factory=dict)

    def pieces(self) -> list:
        b = [0, *self.cuts, len(self.body)]
        return [self.body[b[i]:b[i + 1]] for i in range(len(b) - 1)]


def carried(label: str, R: bytes, t: int, **meta) -> Case:
    """R whose first t bytes (an unterminated line start) are the carried tail: batch 0 holds complete lines, batch 1 those t
    bytes alone, batch 2 the rest of R."""
    assert b"\n" not in R[:t]
    return Case(label, FIRST + R, (len(FIRST), len(FIRST) + t), dict(t=t, **meta))


# ------------------------------------------------------------------ produce kernel
CARRIES = list(range(0, 49)) + list(range(BUF - 48, BUF + 1))


def produce_carry_cases() -> list:
    """A carried tail of t bytes, the '\\n' of the line it starts at window offset o (8160..8200: o >= BUF is the next window)."""
    out = []
    for t in CARRIES:
        A = r16(t)
        for o in range(BUF - 32, BUF + 9):
            p = o - (A - t)                   # R position of the '\n'
            if p < max(t, MIN_DATA - 1):
                continue
            R = data_line(p + 1) + b"\n" + chunk(b"after") + END
            out.append(carried("produce.window_end", R, t, o=o, nl=p))
    return out


def produce_long_cases() -> list:
    """Lines of BUF-32 .. BUF+16 bytes starting at window offset a = 0..15: the in-window / in-carry-slot threshold."""
    out = []
    for a in range(16):
        for n in range(BUF - 32, BUF + 17):
            body = filler(a) + data_line(n) + chunk(b"next") + END
            out.append(Case("produce.long_threshold", body, (), dict(a=a, n=n, line=(a, a + n))))
    return out


SPLIT_TOKENS = {"nlnl": b"\n\n", "crlf": b"\r\n", "data": b"data: ", "nbsp": "\u00a0".encode(), "ideo": "\u3000".encode()}


def _with_token(name: str, at: int) -> bytes:
    """A stream whose bytes [at, at + len(token)) are the token (at >= MIN_DATA + 8)."""
    tok = SPLIT_TOKENS[name]
    if name == "nlnl":
        return data_line(at + 1) + b"\n" + END
    if name == "crlf":
        return data_line(at + 2, eol=b"\r\n") + b"\r\n" + END
    if name == "data":
        return filler(at) + chunk(b"opened") + END
    # a space Go's strings.TrimSpace removes, alternately after the payload and before "data: "
    if at % 2:
        return filler(at - 300) + data_line(301)[:-1] + tok + b"\n\n" + END
    return filler(at) + tok + chunk(b"spaced") + END


def produce_split_cases() -> list:
    """Each token split at every byte across the end of the first window (carried front t = 0..15, so every alignment) and
    across a batch end (the token at every alignment mod 16)."""
    out = []
    for name, tok in SPLIT_TOKENS.items():
        for j in range(len(tok) + 1):
            for t in range(16):
                at = t + BUF - r16(t) - j
                R = _with_token(name, at)
                assert R[at:at + len(tok)] == tok
                out.append(carried("produce.split_window", R, t, tok=name, j=j, at=at))
                at = 400 + t
                R = _with_token(name, at)
                assert R[at:at + len(tok)] == tok
                c = len(FIRST) + at + j
                out.append(Case("produce.split_batch", FIRST + R, (len(FIRST) + 100, c), dict(tok=name, j=j, at=len(FIRST) + at)))
    return out


def produce_round_cases() -> list:
    """Rounds of 63, 64, 65, 128 and 129 lines in one window; a terminating chunk as line 64 and 65; "[DONE]" lines as the 15th
    to 18th "[DONE]" of a round (DONE_MAX candidates, then the fallback scan)."""
    out = []
    for n in (LT_MAX - 1, LT_MAX, LT_MAX + 1, 2 * LT_MAX, 2 * LT_MAX + 1):
        out.append(Case("produce.rounds", SHORT * n, (), dict(n_lines=n)))
        out.append(Case("produce.rounds", SHORT * (n - 1) + chunk(b"last", eol=b"\n") + END, (), dict(n_lines=n + END.count(b"\n"))))
    for k in (LT_MAX - 1, LT_MAX):
        body = SHORT * k + STOP_LINE + SHORT * 10 + END
        out.append(Case("produce.terminate_round", body, (), dict(line=k)))
    for k in (DONE_MAX - 1, DONE_MAX, DONE_MAX + 1, DONE_MAX + 2):
        for kind in ("content", "exact", "bare"):
            d = {"content": chunk(b"[DONE]", eol=b"\n"), "exact": b"data: [DONE]\n", "bare": b"[DONE]\n"}[kind]
            body = d * (k - 1) + chunk(b"tail [DONE]", eol=b"\n") + SHORT * 3 + d + chunk(b"z") + END
            out.append(Case("produce.done_candidates", body, (), dict(k=k, kind=kind)))
    return out


# ------------------------------------------------------------------ tile kernel: packing (one batch of many connections)
@dataclass
class Batch:
    """Streams of many connections, meant to be submitted together: conn i gets bodies[i]. first_cut: a batch boundary for
    every connection (None: one batch)."""
    label: str
    bodies: list
    first_cut: list | None = None
    meta: dict = field(default_factory=dict)


def sized(n: int, k: int = 0) -> bytes:
    """A stream of exactly n bytes (n >= 16) that ends in complete lines."""
    if n < MIN_DATA + len(END):
        small = b'data: {"choices":[{"index":%d}]}\n\n' % k
        if n >= len(small):
            return small + b"\n" * (n - len(small))
        return (b"data: {}\n" + b"\n" * n)[:n - 1] + b"\n"
    return filler(n - len(END)) + END


def tile_pack_batches() -> list:
    out = []
    for d in (-16, 0, 16):          # regions summing to TILE - 16, TILE, TILE + 16 over three segments
        out.append(Batch("tile.pack_sum", [sized(16384), sized(16384), sized(16384 + d)] + [sized(32, k) for k in range(5)],
                         meta=dict(d=d)))
    for n in (MAX_TSEGS - 1, MAX_TSEGS, MAX_TSEGS + 1, 2 * MAX_TSEGS, 2 * MAX_TSEGS + 1):
        out.append(Batch("tile.pack_count", [sized(16, k) for k in range(n)], meta=dict(n=n)))
    for n in (PLAN_GROUP - 1, PLAN_GROUP, PLAN_GROUP + 1, PLAN_GROUP + 76):
        out.append(Batch("tile.pack_group", [sized(1008, k) for k in range(n)], meta=dict(n=n)))
    for extra in (0, 16):           # a region of exactly TILE stays a tile; 16 bytes more goes to big_segment
        out.append(Batch("tile.pack_whole", [sized(32)] * 3 + [sized(TILE + extra)] + [sized(32)] * 3, meta=dict(extra=extra)))
    # finished connections inside a full tile: every third terminates in batch 0 (mode R); batch 1 has 2 * MAX_TSEGS + 1
    bodies, cuts = [], []
    for k in range(2 * MAX_TSEGS + 1):
        if k % 3 == 0:
            b = chunk(b"a") + chunk(b"end", b'"stop"')
            cuts.append(len(b))
            bodies.append(b + b"data: {}\n\n")
        else:
            b = chunk(b"a")
            cuts.append(len(b))
            bodies.append(b + b"data: {}\n\n")
    out.append(Batch("tile.pack_finished", bodies, cuts))
    return out


# ------------------------------------------------------------------ tile kernel: big_segment
BIG_CARRIES = [0, 1, 15, 16, 17, 1000, BUF - 1, BUF, 20000, 32768 - 200]


def _big_prefix(t: int) -> bytes:
    return data_line(t + 200)


def big_segment_cases() -> list:
    out = []
    for t in BIG_CARRIES:
        head = _big_prefix(t)
        for win in (0, 1):
            for d in (-17, -16, -9, -2, -1, 0, 1):
                # the '\n' of a 600-byte line at window end + d (d = -1: the window's last byte); d <= -2: the next line
                # starts in the last 16 bytes of the window (the `front` path of the next window)
                probe = tile_windows(head[:t], head[t:] + filler(3 * TILE))
                if win == 1:
                    first = probe[0]
                    R0 = head + filler(first.s1 - 700 - len(head)) + data_line(1400)    # an unterminated line across the end
                    probe = tile_windows(R0[:t], R0[t:] + filler(3 * TILE))
                    E = probe[1].s1
                    pre = R0
                else:
                    E = probe[0].s1
                    pre = head
                nl = E + d
                R = pre + filler(nl - 599 - len(pre)) + data_line(600) + filler(TILE + 5000) + END
                out.append(carried("tile.big_window_end", R, t, win=win, d=d, nl=nl))
        if t in (0, 17, 32768 - 200):
            out.append(carried("tile.big_4mib", head + filler(4 << 20) + END, t))
    R = filler(60000) + data_line(TILE + 64) + END
    out.append(Case("tile.big_no_newline", R, (), dict(line=(60000, 60000 + TILE + 64))))
    R = filler(70000) + STOP_LINE + filler(60000) + END
    out.append(Case("tile.big_terminate", R, (), dict(at=70000)))
    R = filler(120000) + b"data: [DONE]\n\n" + filler(30000) + END
    out.append(Case("tile.big_done_exact", R, (), dict(at=120000)))
    return out


# ------------------------------------------------------------------ tile kernel: line rounds and the unquote queue
def tile_round_cases() -> list:
    out = []
    for n in (LCAP - 1, LCAP, LCAP + 1, 2 * LCAP, 2 * LCAP + 1):
        out.append(Case("tile.rounds", SHORT * n + END, (), dict(n_lines=n + END.count(b"\n"))))
    for k in (LCAP - 1, LCAP):
        out.append(Case("tile.terminate_round", SHORT * k + STOP_LINE + SHORT * 20 + END, (), dict(line=k)))
    return out


def tile_round_batches() -> list:
    """Two connections in one tile: the LCAP round boundary inside the second segment, and at the segment boundary."""
    out = []
    for a in (LCAP - 200, LCAP - 1, LCAP, LCAP + 1):
        out.append(Batch("tile.rounds_segments", [SHORT * a, SHORT * 300 + END], meta=dict(a=a)))
        out.append(Batch("tile.rounds_segments", [SHORT * a + STOP_LINE + SHORT * 5, SHORT * 300 + END], meta=dict(a=a)))
    return out


ESC_CONTENT = b'data: {"choices":[{"index":0,"delta":{"content":"a\\nb\\u00e9"},"finish_reason":null}]}\n'
ESC_ARGS = b'data: {"choices":[{"delta":{"tool_calls":[{"index":0,"function":{"arguments":"{\\"k\\":\\"v\\n\\"}"}}]}}]}\n'
DUPS = {
    "content_null": b'data: {"choices":[{"index":0,"delta":{"content":"a\\nb","content":null}}]}\n',
    "content_str": b'data: {"choices":[{"index":0,"delta":{"content":"a\\nb","content":"b"}}]}\n',
    "args_null": b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"function":{"arguments":"x\\ny","arguments":null}}]}}]}\n',
    "args_str": b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"function":{"arguments":"x\\ny","arguments":"b"}}]}}]}\n',
}


def unquote_cases() -> list:
    """Rounds with JQ_CAP - 1 .. JQ_CAP + 1 and 300 strings to unquote; a repeated key after an escaped value around queue
    index JQ_CAP."""
    out = []
    for n in (JQ_CAP - 1, JQ_CAP, JQ_CAP + 1, 300):
        for kind, line in (("content", ESC_CONTENT), ("args", ESC_ARGS)):
            out.append(Case("tile.unquote", line * n + END, (), dict(n_jobs=n, kind=kind)))
    for name, dup in DUPS.items():
        for i in (JQ_CAP - 2, JQ_CAP - 1, JQ_CAP, JQ_CAP + 1):
            esc = ESC_ARGS if name.startswith("args") else ESC_CONTENT
            out.append(Case("tile.unquote_dup", esc * i + dup + esc * 8 + END, (), dict(dup=name, index=i)))
    return out


# ------------------------------------------------------------------ tile kernel: template replay limits
def _tpl_line(n_esc: int, n_keys: int, seed: int = 0, arr: bool = False) -> bytes:
    keys = b"".join(b'"k%d":%d,' % (i, (i * 7 + seed) % 10) for i in range(n_keys)) + (b'"l":[0],' if arr else b"")
    return (b'data: {"id":"x","choices":[{"index":0,"delta":{' + keys + b'"content":"' + b"w\\n" * n_esc +
            b'"},"finish_reason":null}]}\n')


T_HDR, T_LIT_MAX, T_SEG_MAX = 7, 1024, 63     # t_build: header words, literal bytes, structural stops of a template


def template_words(payload: bytes):
    """t_build (sse_fused.cu:956-1050) for a simple line without tool calls or usage: (words its template takes in the store,
    structural stops, wildcards), or None when no template is built. Structural stops are unescaped quotes and '[' outside
    strings; a string value and an integer are wildcards; any other segment of more than 3 bytes goes to the literal pool, and
    so do the bytes around an integer in its segment. A template takes T_HDR + (n_struct + 1) + ceil(literal bytes / 4) + 1
    words. None: more than T_SEG_MAX structural stops, more than REC_MAX wildcards (the recorder marks the line not simple), two
    integers in one segment, a literal segment of more than 255 bytes or more than T_LIT_MAX literal bytes."""
    ns = lit = wild = 0
    in_str, seg_a, i, n = False, 0, 0, len(payload)
    while True:
        while i < n and not (payload[i] == 0x22 or (payload[i] == 0x5B and not in_str)):
            i += 2 if in_str and payload[i] == 0x5C else 1
        q = min(i, n)
        seg = payload[seg_a:q]
        if in_str:
            j = q + 1
            while j < n and payload[j] in b" \t\r\n":
                j += 1
            if j < n and payload[j] == 0x3A:                 # a key: literal
                if len(seg) > 255:
                    return None
                lit += len(seg) if len(seg) > 3 else 0
            else:
                wild += 1
        else:
            ints = [m for m in re.finditer(rb"-?\d+(?![\d.eE])", seg)
                    if m.start() == 0 or seg[m.start() - 1:m.start()] in (b":", b",", b"[", b" ")]
            if len(ints) > 1:
                return None
            if ints:
                wild += 1
                pre, suf = ints[0].start(), len(seg) - ints[0].end()
                if pre > 255 or suf > 255:
                    return None
                lit += pre + suf
            else:
                if len(seg) > 255:
                    return None
                lit += len(seg) if len(seg) > 3 else 0
        if q >= n:
            break
        if ns >= T_SEG_MAX:
            return None
        if payload[q] == 0x22:
            in_str = not in_str
        ns += 1
        seg_a = i = q + 1
    if wild > REC_MAX or lit > T_LIT_MAX or in_str:
        return None
    return T_HDR + ns + 1 + (lit + 3) // 4 + 1, ns, wild


def _wild_line(k: int) -> bytes:
    """A line with k + 1 wildcards: the content and k integers, one per segment (nested arrays: each '[' is a structural
    stop)."""
    arr = b"".join(b"[%d," % i for i in range(k - 1)) + b"[%d" % (k - 1) + b"]" * k
    return b'data: {"choices":[{"delta":{"content":"w"}}],"l":' + arr + b"}\n"


def template_cases() -> list:
    """After a shape is learnt (the same skeleton many times first): lines with W_STOPS - 1 .. W_STOPS + 1 stop bytes;
    T_SEG_MAX - 1 .. T_SEG_MAX + 1 structural stops (t_build builds nothing past T_SEG_MAX = W_STRUCT - 1, so no template has
    W_STRUCT stops and the replay's own W_STRUCT compare never binds: t_build's limit is the seam); REC_MAX - 1 .. REC_MAX + 1
    wildcards; more than NREC new shapes in one round."""
    out = []
    learn = _tpl_line(1, 4) * 200
    base = count_stops(_tpl_line(0, 4)[6:-1])
    for s in (W_STOPS - 1, W_STOPS, W_STOPS + 1):
        line = _tpl_line(s - base, 4)
        out.append(Case("tpl.stops", learn + line * 40 + END, (len(learn),), dict(stops=count_stops(line[6:-1]))))
    base = count_structural(_tpl_line(0, 0)[6:-1])
    for s in (T_SEG_MAX - 1, T_SEG_MAX, T_SEG_MAX + 1):
        arr = (s - base) % 2 == 1                  # "l":[0] adds three structural stops, a key two
        line = _tpl_line(1, (s - base - 3 * arr) // 2, arr=arr)
        out.append(Case("tpl.struct", line * 240 + END, (200 * len(line),), dict(struct=count_structural(line[6:-1]))))
    for w in (REC_MAX - 1, REC_MAX, REC_MAX + 1):
        line = _wild_line(w - 1)
        out.append(Case("tpl.wild", line * 240 + END, (200 * len(line),), dict(wild=w)))
    shapes = b"".join(_tpl_line(1, k, seed) for seed in range(3) for k in range(2 * NREC + 3))
    out.append(Case("tpl.new_shapes", shapes * 4 + END, (), dict(n_shapes=2 * NREC + 3)))
    return out


STORE_SHAPES = 60


def _store_line(shape: int) -> bytes:
    """One of STORE_SHAPES shapes that differ in four long key names: most of each template's words are literal bytes."""
    keys = b"".join(b'"s%03d_%d_%s":%d,' % (shape, k, b"k" * 190, k) for k in range(4))
    return b"data: {" + keys + b'"choices":[{"index":0,"delta":{"content":"w"},"finish_reason":null}]}\n'


def template_store_body(reps: int = 5) -> bytes:
    """The STORE_SHAPES shapes reps times over: one segment larger than a tile, so that one CTA walks it window by window
    and records up to NREC new templates in every round, until the store is full."""
    return b"".join(_store_line(k) for _ in range(reps) for k in range(STORE_SHAPES)) + END


# ------------------------------------------------------------------ line-length limit
def limit_cases(limit: int) -> list:
    """Lines of limit - 1, limit and limit + 1 bytes ('\\n' included), reached four ways: complete inside one segment; completed
    from the carry slot; spread over three batches; inside a big_segment window after the first. Unterminated tails of
    limit - 2 .. limit + 1 bytes, in a segment that fits a tile and at the end of one that does not (big_segment, then
    finish_segment); a carried tail of up to the slot exactly, completed by a segment larger than a tile."""
    out = []
    for n in (limit - 1, limit, limit + 1):
        line = data_line(n)
        body = FIRST + line + chunk(b"after") + END
        s = len(FIRST)
        out.append(Case("limit.one_segment", body, (), dict(n=n, line=(s, s + n))))
        out.append(Case("limit.from_carry", body, (s + n - 700,), dict(n=n, line=(s, s + n))))
        out.append(Case("limit.three_batches", body, (s + 1000, s + n // 2), dict(n=n, line=(s, s + n))))
        pre = filler(TILE + 3000)
        body = pre + line + chunk(b"after") + END
        out.append(Case("limit.big_window", body, (), dict(n=n, line=(len(pre), len(pre) + n))))
        tail = FIRST + line[:-1]                      # an unterminated tail of n - 1 bytes, then n bytes
        out.append(Case("limit.tail", tail, (len(FIRST) + 100,), dict(n=n - 1, line=(len(FIRST), len(tail)))))
        out.append(Case("limit.tail", tail + b"x", (len(FIRST) + 100,), dict(n=n, line=(len(FIRST), len(tail) + 1))))
        # the same tails left by the last window of a segment larger than a tile (big_segment, then finish_segment)
        out.append(Case("limit.big_tail", pre + line[:-1], (), dict(n=n - 1, line=(len(pre), len(pre) + n - 1))))
        out.append(Case("limit.big_tail", pre + line[:-1] + b"x", (), dict(n=n, line=(len(pre), len(pre) + n))))
        # a carried tail of n - 1 bytes (the slot exactly, for n = limit + 1) completed by a segment larger than a tile
        body = FIRST + line + pre + END
        out.append(Case("limit.big_carry", body, (len(FIRST) + n - 1,), dict(n=n, line=(len(FIRST), len(FIRST) + n))))
    return out


def all_cases() -> list:
    """Every single-connection seam stream except the line-length ones (those fail by design, DESIGN.md §5 deviation 3)."""
    return (produce_carry_cases() + produce_long_cases() + produce_split_cases() + produce_round_cases() + big_segment_cases()
            + tile_round_cases() + unquote_cases() + template_cases())
