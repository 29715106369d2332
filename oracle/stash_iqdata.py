"""Restatement of blah2's IQ-data stash (api/stash/iqdata.js) and of what /stash/iqdata sends.  TEST INFRASTRUCTURE
ONLY: written from the JS source's behaviour, not a copy of it.

  iqdata.js:3          nCpi = 20
  iqdata.js:8          output = [] until the first document
  iqdata.js:36-56      on every new document: output = JSON.parse(body); push output.spectrum, output.frequency and
                       output.timestamp onto three arrays, each dropping its oldest entry beyond nCpi; replace those
                       three members of output with the arrays.  JSON.parse throws on a document it rejects (a
                       truncated one) before output is assigned: nothing changes.
  server.js:102-103    res.send(output): Express sends JSON.stringify(output).

So the stash is the newest document's object with its spectrum, frequency and timestamp replaced by those of the
last 20 documents, members in the document's order.  JSON.parse reads numbers as correctly rounded doubles (Python's
float(); integers too, so ``parse_int=float``).  Not restated: the API loses its first document after start, its
100 ms polling skips documents that arrive faster, and after a truncated document blah2's socket text runs into the
next document, so the API loses that one too; every document given to ``push`` is taken.
"""
from __future__ import annotations

import json

from oracle.stash_maxhold import js_number_text, stringify  # noqa: F401  (js_number_text: for the tests)

N_CPI = 20


class Stash:
    """The stash's state: the three held arrays and the output object."""

    def __init__(self):
        self.spectrum, self.frequency, self.timestamp = [], [], []
        self.output = []

    def push(self, doc: bytes):
        """A new IQ-data document (the bytes blah2 sent on its IQ-data socket)."""
        try:
            out = json.loads(doc.decode("ascii"), parse_int=float, parse_float=float)
        except ValueError:
            return
        for name in ("spectrum", "frequency", "timestamp"):
            held = getattr(self, name)
            held.append(out[name])
            if len(held) > N_CPI:
                held.pop(0)
            out[name] = list(held)
        self.output = out

    def send(self) -> bytes:
        """The bytes of GET /stash/iqdata."""
        return stringify(self.output).encode("ascii")
