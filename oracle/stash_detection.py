"""Restatement of blah2's detection stash (api/stash/detection.js) and of what /stash/detection sends.  TEST
INFRASTRUCTURE ONLY: written from the JS source's behaviour, not a copy of it.

  detection.js:3       time = 300 (seconds)
  detection.js:10      output = [] until the first document
  detection.js:38-40   on every new document: detection = JSON.parse(body); map.push(detection).  JSON.parse throws on
                       a document it rejects (a truncated one), before anything changes.
  detection.js:41-51   for (i = 0; i < map.length; i++) { if ((ts - map[i].timestamp)/1000 > time) map.shift();
                       else break; }  -- i advances while the array shifts: the documents at original positions
                       0, 2, 4, ... are tested, and each stale test removes one document from the front.
  detection.js:52-73   output = {timestamp, delay, doppler, snr}: the held documents flattened in order, detection
                       by detection, each detection with its document's timestamp.
  server.js:99-100     res.send(output): Express sends JSON.stringify(output).

ts is the latest timestamp the API saw, which is the new document's timestamp.  JSON.parse reads numbers as
correctly rounded doubles (Python's float(); integers too, so ``parse_int=float``), and the prune's arithmetic is in
doubles.  Not restated: the API loses its first document after start (server.js:31,141), its 100 ms polling skips
documents that arrive faster, and it ignores a timestamp equal to the last one it saw; every document given to
``push`` is taken.
"""
from __future__ import annotations

import json

from oracle.stash_maxhold import js_number_text, stringify  # noqa: F401  (js_number_text: for the tests)

TIME = 300


class Stash:
    """The stash's state: the parsed documents held, and the output object."""

    def __init__(self):
        self.map = []
        self.output = []

    def push(self, doc: bytes):
        """A new detection document (the bytes blah2 sent on its detection socket)."""
        try:
            d = json.loads(doc.decode("ascii"), parse_int=float, parse_float=float)
        except ValueError:
            return
        ts = d["timestamp"]
        self.map.append(d)
        i = 0
        while i < len(self.map):
            if (ts - self.map[i]["timestamp"]) / 1000 > TIME:
                self.map.pop(0)
            else:
                break
            i += 1
        out = {"timestamp": [], "delay": [], "doppler": [], "snr": []}
        for m in self.map:
            for j in range(len(m["delay"])):
                out["delay"].append(m["delay"][j])
                out["doppler"].append(m["doppler"][j])
                out["snr"].append(m["snr"][j])
                out["timestamp"].append(m["timestamp"])
        self.output = out

    def send(self) -> bytes:
        """The bytes of GET /stash/detection."""
        return stringify(self.output).encode("ascii")
