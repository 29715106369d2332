"""A pipeline's last CPI as blah2's process thread publishes it: fetch() and then every product, in blah2's order."""
import struct

from blah2_b200 import capi


def code(f):
    """f(), or the return code of the B200ddError it raised."""
    try:
        return f()
    except capi.B200ddError as e:
        return e.code


def fetch_result(pipe):
    """Pipeline.fetch() as bytes: (skipped, noisePower and maxPower, the detections' delay, Doppler and SNR)."""
    r = pipe.fetch()
    d = r["detections"]
    return (r["skipped"], struct.pack("<2d", r["noisePower"], r["maxPower"]), d.delay.tobytes(), d.doppler.tobytes(),
            d.snr.tobytes())


def cpi_products(pipe, ts, fetch=fetch_result):
    """[("fetch", fetch(pipe)), ("map", ...), ...]: the CPI's fetch, then its map document, spectrum, max-hold
    document, detection document and stash, IQ-data document and stash and track document at timestamp ts, each as
    its bytes or the return code that refused it."""
    out = [("fetch", fetch(pipe))]
    for name, f in (("map", lambda: pipe.fetch_map_json(ts)),
                    ("spectrum", lambda: pipe.fetch_spectrum().tobytes()),
                    ("maxhold", lambda: pipe.fetch_maxhold(ts)),
                    ("detection", lambda: pipe.fetch_detection_json(ts)),
                    ("detection_stash", pipe.fetch_detection_stash),
                    ("iqdata", lambda: pipe.fetch_iqdata_json(ts)),
                    ("iqdata_stash", pipe.fetch_iqdata_stash),
                    ("track", lambda: pipe.fetch_track_json(ts))):
        out.append((name, code(f)))
    return out
