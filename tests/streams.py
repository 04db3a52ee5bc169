"""Upstream bodies shared by the GPU tests: chat.completion.chunk events, lines longer than the carry slot (which continue in
the line pool), and filler payloads dealt over many connections to put a decode launch in a chosen shape."""
import numpy as np

from tests.corpus import _plain

SLOT = 32768                # the carry slot of the line-pool tests
PAGE = 65536                # their line-pool page
FILLER_CONNS = 4096         # the connections dealt() spreads payloads over


def chunk(content, fin="null"):
    return b'data: {"choices":[{"index":0,"delta":{"content":"%s"},"finish_reason":%s}]}\n\n' % (content, fin.encode())


USAGE = b'data: {"choices":[],"usage":{"prompt_tokens":11,"completion_tokens":22,"total_tokens":33}}\n\n'
UNITS = [b"ab", b"cdef", b"\\n", b'\\"', b"\\\\", b"\\u00e9", "é".encode(), "€".encode(), "😀".encode(), b"\\t", b" "]


def filler(rng, n):
    """n bytes of a JSON string body: escapes and multi-byte UTF-8 mixed into ASCII."""
    parts, k = [], 0
    idx = rng.integers(0, len(UNITS), size=n // 2 + 8)
    for i in idx:
        u = UNITS[i]
        if k + len(u) > n - 6:
            break
        parts.append(u)
        k += len(u)
    parts.append(b"x" * (n - k))
    return b"".join(parts)


def _ascii_args(rng, n):
    """JSON text of n bytes, escaped as a JSON string body (a file written whole through an MCP tool)."""
    head = b'{\\"path\\":\\"notes.md\\",\\"content\\":\\"'
    tail = b'\\"}'
    line = b"line of the file\\n"
    body = (line * ((n - len(head) - len(tail)) // len(line) + 1))[:n - len(head) - len(tail)]
    if body.endswith(b"\\"):
        body = body[:-1] + b"x"
    return head + body + tail


def long_line(kind, n, rng):
    """One line of exactly n bytes ('\\n' or '\\r\\n' included)."""
    end = b"\r\n" if kind == "crlf" else b"\n"
    if kind in ("toolcall", "terminal"):
        fin = b'"tool_calls"' if kind == "terminal" else b"null"
        pre = b'data: {"choices":[{"index":0,"delta":{"tool_calls":[{"index":0,"id":"call_big","type":"function","function":{"name":"write_file","arguments":"'
        post = b'"}}]},"finish_reason":' + fin + b"}]}" + end
        return pre + _ascii_args(rng, n - len(pre) - len(post)) + post
    pre = b'data: {"id":"c","choices":[{"index":0,"delta":{"content":"'
    post = b'"},"finish_reason":null}]}' + end
    body = filler(rng, n - len(pre) - len(post))
    if kind == "done":       # "[DONE]" inside the line: mode R swallows it (agent.go:181-184), it is still decoded
        mid = len(body) // 2
        while body[mid - 1:mid] == b"\\" or (body[mid] & 0xC0) == 0x80:
            mid += 1
        body = body[:mid] + b"[DONE]" + body[mid + 6:]
    return pre + body + post


def stream_with(line, kind):
    body = chunk(b"Hello") + chunk(b"world") + line + (b"\r\n" if kind == "crlf" else b"\n")
    if kind == "terminal":    # the long line itself ends the agent loop: what follows is never read in mode R
        return body + chunk(b"never read") + b"data: [DONE]\n\n"
    return body + chunk(b"bye", '"stop"') + USAGE + b"data: [DONE]\n\n"


def burst(n, rng, size=200_000, kinds=("toolcall", "content", "terminal")):
    """n streams, each with one long line of about `size` bytes (1,009 more per stream), its kind taken from kinds in turn."""
    return [stream_with(long_line(kinds[i % len(kinds)], size + 1009 * i, rng), kinds[i % len(kinds)]) for i in range(n)]


def holder(rng, size, kind="toolcall"):
    """A stream with a long line, and where to cut it so that its connection holds `size // 2` bytes of that line in pages."""
    body = stream_with(long_line(kind, size, rng), kind)
    return body, len(chunk(b"Hello")) + len(chunk(b"world")) + size // 2


def filler_payload(kind: str, n: int) -> bytes:
    """A valid chunk of about n bytes: "strings" carries them in a plain content string. "nostring" is exactly n bytes of a
    number array under a key the decoder does not know (below 16 bytes: a number), so its lane is never inside a string."""
    if kind == "strings":
        head, tail = b'{"choices":[{"index":0,"delta":{"content":"', b'"},"finish_reason":null}]}'
        return head + _plain(max(1, n - len(head) - len(tail))) + tail
    if n < 16:
        return b"1" * n
    nums = (b"1234567," * (n // 8))[:n - 15]
    return b'{"x_filler":[' + (nums[:-1] + b"8" if nums.endswith(b",") else nums) + b"]}"


def dealt(per_batch):
    """per_batch[b]: the payloads micro-batch b carries, dealt over FILLER_CONNS connections as "data: " events. Returns
    (bodies, bounds, lines): batch b takes exactly connection c's share of per_batch[b]; lines[c] holds (start of the line,
    offset of its '\\n', payload offset, payload length) per data line of body c."""
    pieces = [[pl[c::FILLER_CONNS] for c in range(FILLER_CONNS)] for pl in per_batch]
    bodies, bounds, lines = [], [], []
    for c in range(FILLER_CONNS):
        at, row, ents = 0, [0], []
        for p in pieces:
            for pay in p[c]:
                ents.append((at, at + 6 + len(pay), at + 6, len(pay)))
                at += len(pay) + 8
            row.append(at)
        bodies.append(b"".join(b"data: " + pay + b"\n\n" for p in pieces for pay in p[c]))
        bounds.append(row); lines.append(ents)
    return bodies, np.array(bounds, dtype=np.int64), lines
