"""An independent Python model of the reference's streaming path ABOVE json.Unmarshal (which tests/go_model.py models):

  lines()                       providers/core/provider.go:308-341   bufio.ReadBytes('\\n'), unterminated tail dropped
  trim_space()                  strings.TrimSpace (utf8.DecodeRune / DecodeLastRune + unicode.IsSpace), written from the Go docs
  run_with_stream()             mcp/agent.go:169-248                 one agent iteration
  parse_streaming_tool_calls()  mcp/agent.go:377-481
  telemetry()                   api/middlewares/telemetry.go:190-277

Pure Python, statement by statement from the cited Go code, in a different language and shape than oracle/sse_oracle.c;
tests/test_oracle_stream_model.py pins the C oracle against it.
"""
from __future__ import annotations

from tests import go_model as gm

RUNE_ERROR = 0xFFFD
_SPACE = {0x09, 0x0A, 0x0B, 0x0C, 0x0D, 0x20, 0x85, 0xA0, 0x1680, 0x2028, 0x2029, 0x202F, 0x205F, 0x3000} | set(range(0x2000, 0x200B))


def decode_rune(b: bytes, i: int, end: int):
    """utf8.DecodeRune(b[i:end]) -> (rune, size); invalid encodings give (RuneError, 1)."""
    n = end - i
    if n < 1:
        return RUNE_ERROR, 0
    c0 = b[i]
    if c0 < 0x80:
        return c0, 1
    if 0xC2 <= c0 <= 0xDF:
        need, lo, hi, r = 1, 0x80, 0xBF, c0 & 0x1F
    elif 0xE0 <= c0 <= 0xEF:
        need, r = 2, c0 & 0x0F
        lo, hi = (0xA0, 0xBF) if c0 == 0xE0 else (0x80, 0x9F) if c0 == 0xED else (0x80, 0xBF)
    elif 0xF0 <= c0 <= 0xF4:
        need, r = 3, c0 & 0x07
        lo, hi = (0x90, 0xBF) if c0 == 0xF0 else (0x80, 0x8F) if c0 == 0xF4 else (0x80, 0xBF)
    else:
        return RUNE_ERROR, 1
    if n < need + 1:
        return RUNE_ERROR, 1
    c1 = b[i + 1]
    if not lo <= c1 <= hi:
        return RUNE_ERROR, 1
    r = (r << 6) | (c1 & 0x3F)
    for k in range(2, need + 1):
        c = b[i + k]
        if not 0x80 <= c <= 0xBF:
            return RUNE_ERROR, 1
        r = (r << 6) | (c & 0x3F)
    return r, need + 1


def decode_last_rune(b: bytes, start0: int, end: int):
    """utf8.DecodeLastRune(b[start0:end]) -> (rune, size)."""
    if end - start0 == 0:
        return RUNE_ERROR, 0
    start = end - 1
    if b[start] < 0x80:
        return b[start], 1
    lim = max(start0, end - 4)
    start -= 1
    while start >= lim:
        if (b[start] & 0xC0) != 0x80:      # utf8.RuneStart
            break
        start -= 1
    if start < start0:
        start = start0
    r, size = decode_rune(b, start, end)
    if start + size != end:
        return RUNE_ERROR, 1
    return r, size


def trim_space(s: bytes) -> bytes:
    a, e = 0, len(s)
    while a < e:
        r, n = decode_rune(s, a, e)
        if r not in _SPACE:
            break
        a += n
    while e > a:
        r, n = decode_last_rune(s, a, e)
        if r not in _SPACE:
            break
        e -= n
    return s[a:e]


def lines(body: bytes):
    """provider.go:322-334: every '\\n'-terminated line including its '\\n'; the tail is dropped with the read error."""
    out, i = [], 0
    while True:
        j = body.find(b"\n", i)
        if j < 0:
            return out
        out.append(body[i:j + 1])
        i = j + 1


def run_with_stream(body: bytes):
    """agent.go:169-248 for one iteration. Returns dict(frames, builder, content, has_tool_calls, terminated)."""
    frames, builder, content = [], bytearray(), b""
    has_tool_calls = terminated = False
    for line in lines(body):
        trimmed = trim_space(line)
        if b"[DONE]" in trimmed:
            builder += line                                  # :181-184 (the raw line)
            continue
        if not trimmed.startswith(b"data: "):
            continue
        chunk_data = trimmed[6:]
        if chunk_data == b"":
            continue
        formatted = b"data: " + chunk_data + b"\n\n"
        frames.append(formatted)
        builder += formatted
        ck = gm.unmarshal(chunk_data)
        if not ck["json_ok"]:
            continue
        if ck["n_choices"] == 0:
            continue
        if ck["content"] != b"":
            content += ck["content"]
        if ck["tc_nonnil"] and len(ck["tcs"]) > 0:
            for t in ck["tcs"]:
                if t["id"] is not None or (t["function"] and (t["name"] != b"" or t["args"] != b"")):
                    has_tool_calls = True
                    break
        if ck["finish"] in (gm.FIN["stop"], gm.FIN["tool_calls"]):
            terminated = True
            break
    return dict(frames=frames, builder=bytes(builder), content=content, has_tool_calls=has_tool_calls, terminated=terminated)


def _merge(chunks, temp_redecode: bool):
    m = {}
    for ck in chunks:
        if not ck["json_ok"] or ck["n_choices"] == 0 or not ck["tc_nonnil"]:
            continue
        for t in ck["tcs"]:
            idx = t["index"]
            tc = m.setdefault(idx, dict(id=b"", type=b"function", name=b"", args=b""))
            if t["id"] is not None:
                tc["id"] = t["id"]
            if temp_redecode:
                if t["type"] is not None:
                    tc["type"] = t["type"]
                if t["function"]:
                    # agent.go:432-466: the chunk is decoded a second time and EVERY element with this index contributes
                    for u in ck["tcs"]:
                        if u["index"] == idx:
                            if u["name"] != b"":
                                tc["name"] = u["name"]
                            if u["args"] != b"":
                                tc["args"] += u["args"]
            elif t["function"]:
                if t["name"] != b"":
                    tc["name"] = t["name"]
                if t["args"] != b"":
                    tc["args"] += t["args"]
    return m


def parse_streaming_tool_calls(builder: bytes):
    chunks = []
    for line in builder.split(b"\n"):
        line = trim_space(line)
        if line.startswith(b"data: "):
            data = line[6:]
        elif line != b"" and line != b"[DONE]":
            data = line
        else:
            continue
        if data == b"[DONE]" or data == b"":
            break
        chunks.append(gm.unmarshal(data))
    m = _merge(chunks, True)
    return [m[i] for i in range(len(m)) if i in m]


def decoded_payloads(body: bytes, mode_r: bool):
    """The bytes each decoded line hands to json.Unmarshal, in line order. Mode R (agent.go:169-248 up to the terminating
    chunk): an emitted line's chunk_data; a swallowed line containing "[DONE]" as parseStreamingToolCalls (:385-402) sees it,
    the trimmed line without its "data: " prefix, or the bare trimmed line. Mode P with parsing: line[6:len-1] of every line
    that starts with "data: " (the telemetry tap's per-line decode)."""
    if not mode_r:
        return [line[6:-1] for line in lines(body) if line.startswith(b"data: ")]
    out = []
    for line in lines(body):
        trimmed = trim_space(line)
        if b"[DONE]" in trimmed:
            out.append(trimmed[6:] if trimmed.startswith(b"data: ") else trimmed)
            continue
        if not trimmed.startswith(b"data: ") or trimmed[6:] == b"":
            continue
        out.append(trimmed[6:])
        ck = gm.unmarshal(trimmed[6:])
        if ck["json_ok"] and ck["n_choices"] > 0 and ck["finish"] in (gm.FIN["stop"], gm.FIN["tool_calls"]):
            break
    return out


def telemetry(body: bytes):
    pieces = body.split(b"\n\n")
    usage = (0, 0, 0)
    for p in (pieces[-4:] if len(pieces) > 4 else pieces):
        if p == b"" or not p.startswith(b"data: "):
            continue
        p = p[6:]
        if p == b"[DONE]":
            continue
        ck = gm.unmarshal(p)
        if ck["json_ok"] and ck["usage"] is not None:
            usage = ck["usage"]
    chunks = []
    for p in pieces:
        if not p.startswith(b"data: "):
            continue
        p = p[6:]
        if p == b"[DONE]" or p == b"":
            continue
        chunks.append(gm.unmarshal(p))
    m = _merge(chunks, False)
    calls = [m[i] for i in range(len(m)) if i in m and m[i]["name"] != b""]
    return usage, calls
