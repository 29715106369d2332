"""Restatement of blah2's timing stash (api/stash/timing.js) and of what /stash/timing sends.  TEST INFRASTRUCTURE
ONLY: written from the JS source's behaviour, not a copy of it.

  timing.js:3          nCpi = 20
  timing.js:6          output = {} until the first document
  timing.js:32-44      on every new document: cpi = JSON.parse(body); for every key of cpi except "uptime" and "nCpi"
                       (the document has no "uptime", so timestamp, uptime_s and uptime_days are kept), in the
                       document's order: create output[key] = [] when it is new, push cpi[key], drop the oldest entry
                       beyond nCpi.  A document JSON.parse rejects changes nothing.
  server.js:105-106    res.send(output): Express sends JSON.stringify(output): keys in insertion (first-seen) order.

JSON.parse reads numbers as correctly rounded doubles (Python's float(); integers too, so ``parse_int=float``).  Not
restated, as for the other stashes: the API loses its first document after start, and its 100 ms polling skips
documents that arrive faster; every document given to ``push`` is taken.
"""
from __future__ import annotations

import json

from oracle.stash_maxhold import js_number_text, stringify  # noqa: F401  (js_number_text: for the tests)

N_CPI = 20
SKIP = ("uptime", "nCpi")


class Stash:
    """The stash's state: the output object, one array per key."""

    def __init__(self):
        self.output = {}

    def push(self, doc: bytes):
        """A new timing document (the bytes blah2 sent on its timing socket)."""
        try:
            cpi = json.loads(doc.decode("ascii"), parse_int=float, parse_float=float)
        except ValueError:
            return
        for key, v in cpi.items():
            if key in SKIP:
                continue
            held = self.output.setdefault(key, [])
            held.append(v)
            if len(held) > N_CPI:
                held.pop(0)

    def send(self) -> bytes:
        """The bytes of GET /stash/timing."""
        return stringify(self.output).encode("ascii")
