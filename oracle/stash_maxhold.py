"""Restatement of blah2's max-hold stash (api/stash/maxhold.js) and of what /stash/map sends.  TEST INFRASTRUCTURE
ONLY: written from the JS source's behaviour, not a copy of it.

  maxhold.js:3        nCpi = 20
  maxhold.js:54-59    on every new map document: maxhold = JSON.parse(body); map.push(maxhold.data); drop the oldest
                      array beyond nCpi; maxhold.data = process(map).  A document JSON.parse rejects changes nothing.
  maxhold.js:18-35    process(): per cell, Math.max over the held arrays, row and column counts of the oldest one.
  server.js:96-97     res.send(object): Express sends JSON.stringify(object) (no `json spaces` setting): members in
                      insertion order, no whitespace, every number as ECMAScript Number::toString.

JSON.parse reads numbers as correctly rounded doubles, which is Python's float(); integers are doubles too, so
``parse_int=float``.  The stash's first document after the API starts is lost in blah2 (server.js:30,125: the map
listener's buffer starts as `undefined`), and its 100 ms polling skips documents that arrive faster; neither is
restated: every document given to ``push`` is taken.
"""
from __future__ import annotations

import functools
import json

N_CPI = 20


@functools.lru_cache(maxsize=1 << 20)  # map cells repeat their values: k / 100 for an integer k
def js_number_text(d: float) -> str:
    """ECMA-262 Number::toString(d) (radix 10) of a finite double."""
    if d != d or d in (float("inf"), float("-inf")):
        raise ValueError("JSON has no text for a non-finite number")
    if d == 0.0:
        return "0"  # -0 too
    if d < 0:
        return "-" + js_number_text(-d)
    # shortest digits s that read back to d, nearest to d among them (Python's repr rule), and n with
    # d = 0.s * 10^n
    mant, _, exp = ("%r" % d).partition("e")
    ip, _, fp = mant.partition(".")
    digits = (ip + fp).lstrip("0")
    n = len(ip) - (len(ip + fp) - len((ip + fp).lstrip("0"))) + (int(exp) if exp else 0)
    s = digits.rstrip("0")
    k = len(s)
    if k <= n <= 21:
        return s + "0" * (n - k)
    if 0 < n <= 21:
        return s[:n] + "." + s[n:]
    if -6 < n <= 0:
        return "0." + "0" * (-n) + s
    e = n - 1
    sign = "+" if e >= 0 else "-"
    return (s if k == 1 else s[0] + "." + s[1:]) + "e" + sign + str(abs(e))


def stringify(v) -> str:
    """JSON.stringify for what JSON.parse of a map document yields: objects, arrays and numbers."""
    if isinstance(v, dict):
        return "{" + ",".join(json.dumps(k) + ":" + stringify(x) for k, x in v.items()) + "}"
    if isinstance(v, list):
        return "[" + ",".join(stringify(x) for x in v) + "]"
    return js_number_text(float(v))


class Stash:
    """The stash's state: the held `data` arrays and the latest parsed document."""

    def __init__(self):
        self.held = []
        self.maxhold = None

    def push(self, doc: bytes):
        """A new map document (the text blah2 sent on its map socket)."""
        m = json.loads(doc.decode("ascii"), parse_int=float, parse_float=float)
        self.held.append(m["data"])
        if len(self.held) > N_CPI:
            self.held.pop(0)
        # per cell, the maximum over the held arrays (all of one shape)
        m["data"] = [[max(cell) for cell in zip(*rows)] for rows in zip(*self.held)]
        self.maxhold = m

    def send(self) -> bytes:
        """The bytes of GET /stash/map."""
        return stringify(self.maxhold).encode("ascii")
