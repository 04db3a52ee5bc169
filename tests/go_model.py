"""An independent Python model of `json.Unmarshal(data, &types.CreateChatCompletionStreamResponse)`.

Used to pin the C oracle (tests/test_oracle_json.py): syntax acceptance comes from CPython's json module
(RFC 8259, strict control characters, NaN/Infinity rejected), the typed decode below is written from the Go
documentation of encoding/json v1 (decode.go: literalStore / object / array / indirect) and the struct tags of
providers/types/common_types.go -- in a different language and shape than oracle/sse_oracle.c.
"""
from __future__ import annotations

import json

FIN = {"": 0, "stop": 1, "tool_calls": 2, "length": 3, "content_filter": 4, "function_call": 5}


class Num:
    def __init__(self, text):
        self.text = text


class Obj:
    def __init__(self, pairs):
        self.pairs = pairs


def _reject(_):
    raise ValueError("NaN/Infinity are not JSON")


def parse(payload: bytes):
    """Returns (ok, value). Invalid UTF-8 bytes become lone surrogates (Go turns them into U+FFFD later)."""
    try:
        s = payload.decode("utf-8", errors="surrogateescape")
        v = json.loads(s, parse_int=Num, parse_float=Num, parse_constant=_reject,
                       object_pairs_hook=Obj, strict=True)
        return True, v
    except (ValueError, RecursionError):
        return False, None


def go_bytes(s: str) -> bytes:
    """Go's unquote result as bytes: lone surrogates / invalid bytes -> U+FFFD."""
    out = bytearray()
    for ch in s:
        o = ord(ch)
        out += b"\xef\xbf\xbd" if 0xD800 <= o <= 0xDFFF else ch.encode("utf-8")
    return bytes(out)


def fold(s: str) -> str:
    out = []
    for ch in s:
        if "a" <= ch <= "z":
            ch = ch.upper()
        elif ch == "ſ":
            ch = "S"
        elif ch == "K":
            ch = "K"
        out.append(ch)
    return "".join(out)


def _field(fields: dict, key: str):
    k = go_bytes(key).decode("utf-8")     # invalid input became U+FFFD before the lookup
    if k in fields:
        return fields[k]
    fk = fold(k)
    for name, spec in fields.items():
        if fold(name) == fk:
            return spec
    return None


class TypeErr(Exception):
    pass


class Decoder:
    def __init__(self):
        self.err = False

    # -- leaf helpers: return (assigned?, value)
    def string(self, v):
        if v is None:
            return False, None
        if isinstance(v, str):
            return True, go_bytes(v)
        self.err = True
        return False, None

    def integer(self, v):
        if v is None:
            return False, None
        if isinstance(v, Num) and not isinstance(v, bool):
            t = v.text
            body = t[1:] if t.startswith("-") else t
            if body.isdigit():
                n = int(t)
                if -(1 << 63) <= n < (1 << 63):
                    return True, n
        self.err = True
        return False, None

    def f32(self, v):
        if v is None:
            return
        if isinstance(v, Num):
            from fractions import Fraction
            x = abs(Fraction(v.text)) if "e" not in v.text.lower() else abs(_frac(v.text))
            if x >= Fraction(2) ** 128 - Fraction(2) ** 103:
                self.err = True
            return
        self.err = True

    def skip_ok(self, v):
        return

    # -- structs
    def usage(self, v, cur):
        if v is None:
            return None
        if not isinstance(v, Obj):
            self.err = True
            return cur
        u = dict(cur) if cur else dict(prompt=0, completion=0, total=0)
        for k, x in v.pairs:
            f = _field({"completion_tokens": "completion", "prompt_tokens": "prompt", "total_tokens": "total"}, k)
            if f:
                ok, n = self.integer(x)
                if ok:
                    u[f] = n
        return u

    def google(self, v):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        last = None
        seen = False
        for k, x in v.pairs:
            if go_bytes(k) == b"thought_signature":
                seen, last = True, x
        if seen and not (last is None or isinstance(last, str)):
            self.err = True

    def extra(self, v):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        for k, x in v.pairs:
            if _field({"google": 1}, k):
                self.google(x)

    def function(self, v, tc):
        if v is None:
            tc["function"] = False
            tc["name"] = tc["args"] = b""
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        tc["function"] = True
        for k, x in v.pairs:
            f = _field({"arguments": "args", "name": "name"}, k)
            if f:
                ok, s = self.string(x)
                if ok:
                    tc[f] = s

    def tool_call(self, v):
        tc = dict(index=0, id=None, type=None, function=False, name=b"", args=b"")
        if v is None:
            return tc
        if not isinstance(v, Obj):
            self.err = True
            return tc
        for k, x in v.pairs:
            f = _field({"extra_content": "extra", "function": "function", "id": "id", "index": "index", "type": "type"}, k)
            if f == "extra":
                self.extra(x)
            elif f == "function":
                self.function(x, tc)
            elif f in ("id", "type"):
                if x is None:
                    tc[f] = None
                else:
                    ok, s = self.string(x)
                    if ok:
                        tc[f] = s
            elif f == "index":
                ok, n = self.integer(x)
                if ok:
                    tc["index"] = n
        return tc

    def toplp(self, v, with_top):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        names = {"bytes": "bytes", "logprob": "logprob", "token": "token"}
        if with_top:
            names["top_logprobs"] = "top"
        for k, x in v.pairs:
            f = _field(names, k)
            if f == "bytes":
                if x is None:
                    continue
                if not isinstance(x, list):
                    self.err = True
                    continue
                for e in x:
                    self.integer(e)
            elif f == "logprob":
                self.f32(x)
            elif f == "token":
                self.string(x)
            elif f == "top":
                self.lp_list(x, False)

    def lp_list(self, v, with_top):
        if v is None:
            return
        if not isinstance(v, list):
            self.err = True
            return
        for e in v:
            self.toplp(e, with_top)

    def logprobs(self, v):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        for k, x in v.pairs:
            if _field({"content": 1, "refusal": 1}, k):
                self.lp_list(x, True)

    def delta(self, v, st):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        for k, x in v.pairs:
            f = _field({"content": "content", "reasoning": "ps", "reasoning_content": "ps", "refusal": "ps",
                        "role": "s", "tool_calls": "tc"}, k)
            if f == "content":
                ok, s = self.string(x)
                if ok:
                    st["content"] = s
            elif f in ("ps", "s"):
                self.string(x)
            elif f == "tc":
                if x is None:
                    st["tc_nonnil"] = False
                    st["tcs"] = []
                elif not isinstance(x, list):
                    self.err = True
                else:
                    st["tc_nonnil"] = True
                    st["tcs"] = [self.tool_call(e) for e in x]   # (duplicate key: replace, see DESIGN.md)

    def choice(self, v, st):
        if v is None:
            return
        if not isinstance(v, Obj):
            self.err = True
            return
        for k, x in v.pairs:
            f = _field({"delta": "delta", "finish_reason": "fin", "index": "index", "logprobs": "lp"}, k)
            if f == "delta":
                self.delta(x, st)
            elif f == "fin":
                ok, s = self.string(x)
                if ok:
                    st["finish"] = FIN.get(s.decode("utf-8", "replace"), 7)
            elif f == "index":
                self.integer(x)
            elif f == "lp":
                self.logprobs(x)

    def root(self, v):
        res = dict(n_choices=0, usage=None, st=self._fresh())
        if v is None:
            return res
        if not isinstance(v, Obj):
            self.err = True
            return res
        for k, x in v.pairs:
            f = _field({"choices": "choices", "created": "int", "id": "s", "model": "s", "object": "s",
                        "reasoning_format": "s", "system_fingerprint": "s", "usage": "usage"}, k)
            if f == "choices":
                if x is None:
                    res["n_choices"] = 0
                    res["st"] = self._fresh()
                elif not isinstance(x, list):
                    self.err = True
                else:
                    res["n_choices"] = len(x)
                    if not x:              # decode.go array(): [] sets a fresh slice of capacity 0; a later array starts anew
                        res["st"] = self._fresh()
                    for i, e in enumerate(x):
                        self.choice(e, res["st"] if i == 0 else self._fresh())
            elif f == "int":
                self.integer(x)
            elif f == "s":
                self.string(x)
            elif f == "usage":
                res["usage"] = self.usage(x, res["usage"])
        return res

    @staticmethod
    def _fresh():
        return dict(content=b"", finish=0, tc_nonnil=False, tcs=[])


def _frac(text):
    from fractions import Fraction
    t = text.lower()
    m, e = t.split("e")
    e = int(e)
    if e > 5000:
        return Fraction(0) if Fraction(m) == 0 else Fraction(10) ** 5000
    if e < -5000:
        return Fraction(0)
    return Fraction(m) * (Fraction(10) ** e)


def unmarshal(payload: bytes) -> dict:
    """Same dictionary shape as tests.util.chunk_to_dict."""
    ok, v = parse(payload)
    if not ok:
        return dict(json_ok=False)
    d = Decoder()
    res = d.root(v)
    if d.err:
        return dict(json_ok=False)
    out = dict(json_ok=True, n_choices=min(res["n_choices"], 0xFFFF), finish=0, usage=None, content=b"",
               tc_nonnil=False, tc_valid=False, tcs=[])
    if res["usage"] is not None:
        u = res["usage"]
        out["usage"] = (u["prompt"], u["completion"], u["total"])
    if res["n_choices"] > 0:
        st = res["st"]
        out["finish"] = st["finish"]
        out["content"] = st["content"]
        out["tc_nonnil"] = st["tc_nonnil"]
        out["tcs"] = st["tcs"]
        out["tc_valid"] = any(t["id"] is not None or (t["function"] and (t["name"] or t["args"])) for t in st["tcs"])
    return out


DEPTH_LIMIT = 128


def depth_limited(payload: bytes, limit: int = DEPTH_LIMIT) -> bool:
    """The product's documented nesting limit (DESIGN.md §5, deviation 2), restated independently of oracle/sse_oracle.c: True
    when a container opens while `limit` are open, before the payload's first syntax error. The error position is the one
    CPython's json reports; depth is a bracket count outside strings up to it. Payloads with NaN / Infinity literals (which
    CPython reports without a position) are outside this model."""
    s = payload.decode("utf-8", errors="surrogateescape")
    try:
        json.loads(s, object_pairs_hook=Obj, strict=True)
        err = len(s)
    except json.JSONDecodeError as e:
        err = e.pos
    assert "NaN" not in s and "Infinity" not in s
    depth, in_str, esc = 0, False, False
    for ch in s[:err]:
        if in_str:
            if esc:
                esc = False
            elif ch == "\\":
                esc = True
            elif ch == '"':
                in_str = False
        elif ch == '"':
            in_str = True
        elif ch in "[{":
            if depth >= limit:
                return True
            depth += 1
        elif ch in "]}":
            depth -= 1
    return False
