"""The reference's own Preprocess::process (oracle/_ref/libpreprocess_ref.so), live or replayed, in the scheme of
tests/refcalls.py: where oracle/_ref is built, RefPreprocess runs it and checks each answer against
tests/golden/ref/<key>.npz; with FASTLIO_RECORD_REF=DIR it writes the answers to DIR/<key>.npz instead; where oracle/_ref is
not built, it replays the stored answers.  Answers are stored under a digest of the call's inputs, so a call whose inputs
change finds no answer and fails instead of reading another call's.

An answer is (|pl_surf|, digest of the xyzi bytes, digest of the curvature bytes, pl_surf.back().curvature) and, for calls
made with keep_ms (the Velodyne yaw path, whose times the device reproduces within a bound rather than bit for bit), the
curvature array itself.
"""
import os
import warnings

import numpy as np
import pytest

from oracle import preprocess_ref
from refcalls import GOLD, digest


class RefPreprocess:
    def __init__(self, key: str):
        self.key, self.rec = key, {}
        path = os.path.join(GOLD, key + ".npz")
        self.record_dir = os.environ.get("FASTLIO_RECORD_REF")
        self.live = preprocess_ref.available()
        if self.record_dir:
            assert self.live, "recording needs oracle/_ref"
            self.stored = None
        elif os.path.exists(path):
            with np.load(path) as g:
                self.stored = dict(g)
        elif not self.live:
            pytest.fail(f"no reference answers: neither oracle/_ref nor {path}")
        else:
            self.stored = None

    def process(self, raw, offsets, lidar_type, n_scans, scan_rate, time_unit, pfn, blind, keep_ms=False):
        """-> dict(count, xyzi_digest, ms_digest, last_ms[, ms]); with the live reference also xyzi and ms."""
        params = np.array([lidar_type, n_scans, scan_rate, time_unit, pfn, int(keep_ms)], np.int64)
        tag = "p" + digest(np.ascontiguousarray(raw).view(np.uint8), np.asarray(offsets, np.int32), params, np.float64(blind))
        full = None
        out = None
        if self.live:
            xyzi, ms = preprocess_ref.process(raw, offsets, lidar_type, n_scans, scan_rate, time_unit, pfn, blind)
            full = (xyzi, ms)
            out = (np.int64(len(ms)), np.bytes_(digest(xyzi)), np.bytes_(digest(ms)), np.float32(ms[-1] if len(ms) else 0.0))
            if keep_ms:
                out = out + (ms,)
        if self.stored is not None:
            if f"{tag}_n" not in self.stored:
                why = f"{self.key}: a call with inputs {tag} was not recorded"
                if out is None:
                    pytest.fail(why + "; record the answers again (FASTLIO_RECORD_REF)")
                warnings.warn(why + "; judged by the live reference only")
            else:
                want = tuple(self.stored[f"{tag}_o{j}"] for j in range(int(self.stored[f"{tag}_n"])))
                if out is None:
                    out = want
                else:
                    assert all(np.array_equal(a, b) for a, b in zip(out, want)), f"{self.key}: {tag} differs from the stored answer"
        if self.record_dir:
            self.rec[f"{tag}_n"] = np.int32(len(out))
            for j, o in enumerate(out):
                self.rec[f"{tag}_o{j}"] = o
            os.makedirs(self.record_dir, exist_ok=True)
            np.savez_compressed(os.path.join(self.record_dir, self.key + ".npz"), **self.rec)
        r = dict(count=int(out[0]), xyzi_digest=out[1].item().decode(), ms_digest=out[2].item().decode(), last_ms=np.float32(out[3]))
        if keep_ms:
            r["ms"] = np.asarray(out[4], np.float32)
        if full is not None:
            r["xyzi"], r["ms_full"] = full
        return r
