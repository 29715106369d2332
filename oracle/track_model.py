"""CPU model of the device tracker: blah2's Tracker::process + Track::to_json (src/process/tracker/Tracker.cpp,
src/data/Track.cpp) restated in the parallel form blah2_b200/csrc/tracker.cu computes (DESIGN.md §9).
TEST INFRASTRUCTURE ONLY.

Per CPI with n0 tracks at entry:
  a      = whether j* exists, the first detection with -1 < delay < 1 and -(1/cpi) < doppler < 1/cpi (association
           compares against delay 0, Doppler 0, not against the prediction);
  D[i]   = ((a ? 0 : c[i]) + 1 > nDelete) for positions i < n0 (c = the per-position inactivity counters);
  r      = the exclusive prefix sum of D;
  iteration i runs iff i + r[i] < n0: it sets c[i] = (a ? 0 : c[i]) + 1 and processes the track at ORIGINAL index
  i + r[i]; the originals at {i : iteration i runs and D[i]} are removed; survivors keep their order.
Then every unassociated detection starts 2 nAcc + 1 tentative tracks.  Numbers are written by the product's host
formatter (capi.format_track_doubles: Writer::Double at two decimal places, checked against rapidjson elsewhere).
"""
from __future__ import annotations

import numpy as np

C_LIGHT = 299792458
MAX_INDEX = 65535
TENTATIVE, ASSOCIATED, ACTIVE, COASTING = 0, 1, 2, 3
NAMES = ("TENTATIVE", "ASSOCIATED", "ACTIVE", "COASTING")
U64 = 1 << 64


def hypotheses(cpi, maxAcc):
    """accInit of Tracker::Tracker, or None where (int)maxAcc or the uint16_t conversion is undefined."""
    cpi, maxAcc = float(cpi), float(maxAcc)
    if not (-2147483649.0 < maxAcc < 2147483648.0):
        return None
    with np.errstate(divide="ignore", invalid="ignore", over="ignore"):
        res = float(np.float64(1.0) / (np.float64(cpi) * np.float64(cpi)))
        q = float(np.float64(float(int(maxAcc))) / np.float64(res))
    if not (-1.0 < q < 65536.0):
        return None
    n_acc = int(q)
    return [res * (i - n_acc) for i in range(2 * n_acc + 1)]


class TrackModel:
    def __init__(self, m, n, nDelete, cpi, maxAcc, fs, fc):
        self.m, self.n, self.n_delete = int(m), int(n), int(nDelete)
        self.acc_init = hypotheses(cpi, maxAcc)
        assert self.acc_init is not None
        inv = 1.0 / float(cpi) if cpi != 0 else float("inf")
        self.dop_lo, self.dop_hi = 0.0 - inv, 0.0 + inv
        self.range_res = C_LIGHT / int(fs)
        self.lam = C_LIGHT / int(fc)
        self.tracks = []  # dicts: id, acc, cur (delay, doppler), hist [(delay, doppler)], states [codes]
        self.counter = []  # per position, never cleared
        self.inext = 0
        self.timestamp = 0

    def _c(self, i):
        while len(self.counter) <= i:
            self.counter.append(0)
        return self.counter[i]

    def _update_track(self, t, assoc, ad, af, T):
        d0, f0 = t["cur"]
        a0 = t["acc"]
        if assoc:
            t["hist"].append((ad, af))
            with np.errstate(all="ignore"):
                t["acc"] = float(np.float64(af - f0) / np.float64(T))
            t["states"].append(ASSOCIATED)
            L = len(t["states"])
            if L >= self.n:
                hits = sum(1 for s in t["states"][L - self.n:] if s in (ACTIVE, ASSOCIATED))
                if hits >= self.m:
                    t["states"][-1] = ACTIVE
        with np.errstate(all="ignore"):
            f0_, a0_, T_ = np.float64(f0), np.float64(a0), np.float64(T)
            pd = float(np.float64(d0) + ((f0_ * T_ * np.float64(self.lam)) + (np.float64(0.5) * a0_ * T_ * T_))
                       / np.float64(self.range_res))
            pf = float(f0_ + a0_ * T_)
        t["cur"] = (pd, pf)
        t["hist"].append((pd, pf))
        last = t["states"][-1]
        t["states"].append(COASTING if last == ACTIVE else TENTATIVE if last == ASSOCIATED else last)

    def process(self, delay, doppler, ts):
        delay = [float(x) for x in delay]
        doppler = [float(x) for x in doppler]
        n0 = len(self.tracks)
        skip = None
        if n0 > 0:
            T = float(np.float64(float((int(ts) - self.timestamp) % U64)) / np.float64(1000.0))
            self.timestamp = int(ts)
            js = next((j for j in range(len(delay)) if -1.0 < delay[j] < 1.0
                       and self.dop_lo < doppler[j] < self.dop_hi), None)
            assoc = js is not None
            ad, af = (delay[js], doppler[js]) if assoc else (0.0, 0.0)
            D = np.array([(0 if assoc else self._c(i)) + 1 > self.n_delete for i in range(n0)], dtype=np.int64)
            r = np.concatenate([[0], np.cumsum(D)[:-1]])
            removed = set()
            for i in range(n0):
                if i + r[i] >= n0:
                    break
                self.counter[i] = (0 if assoc else self.counter[i]) + 1
                self._update_track(self.tracks[i + int(r[i])], assoc, ad, af, T)
                if D[i]:
                    removed.add(i)
            self.tracks = [t for i, t in enumerate(self.tracks) if i not in removed]
            skip = js
        else:
            self.timestamp = int(ts)
        for j in range(len(delay)):
            if j == skip:
                continue
            for a in self.acc_init:
                self.tracks.append(dict(id=self.inext, acc=a, cur=(delay[j], doppler[j]),
                                        hist=[(delay[j], doppler[j])], states=[TENTATIVE]))
                self._c(len(self.tracks) - 1)
                self.inext += 1
                if self.inext >= MAX_INDEX:
                    self.inext = 0

    def to_json(self, ts, fmt):
        """Track::to_json(ts) as bytes, or None when a value it holds is not finite (rapidjson stops there).
        fmt(list of doubles) -> list of texts ("" for a non-finite value)."""
        sent = [t for t in self.tracks if t["states"][-1] != TENTATIVE]
        vals = []
        for t in sent:
            vals += [t["cur"][0], t["cur"][1], t["acc"]] + [h[0] for h in t["hist"]] + [h[1] for h in t["hist"]]
        if not all(np.isfinite(vals)):
            return None
        txt = iter(fmt(vals)) if vals else iter(())
        counts = [sum(1 for t in self.tracks if t["states"][-1] == c) for c in range(4)]
        out = [f'{{"timestamp":{int(ts)},"n":{len(self.tracks)},"nTentative":{counts[0]},'
               f'"nAssociated":{counts[1]},"nActive":{counts[2]},"nCoasting":{counts[3]},"data":[']
        for k, t in enumerate(sent):
            L = len(t["hist"])
            d, f, a = next(txt), next(txt), next(txt)
            hd = [next(txt) for _ in range(L)]
            hf = [next(txt) for _ in range(L)]
            out.append(("," if k else "") + f'{{"id":"{t["id"]:04X}","state":"{NAMES[t["states"][-1]]}",'
                       f'"delay":{d},"doppler":{f},"acceleration":{a},"n":{L},'
                       f'"associated_delay":[{",".join(hd)}],"associated_doppler":[{",".join(hf)}],'
                       f'"associated_state":[{",".join(chr(34) + NAMES[s] + chr(34) for s in t["states"])}]}}')
        out.append("]}")
        return "".join(out).encode()
