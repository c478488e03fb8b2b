"""Regenerates tests/golden/prs_scores.npz from the reference's own RDS fixture (run where the reference tree exists; the
GPU box only sees the committed .npz).

  tests/testthat/testdata/scores-PRS.rds  517 x 11 doubles: snp_PRS scores of tests/testthat/test-6-PRS.R:34-44 at the
                                          thresholds seq(0, 5, by = 0.5)

RDS = gzip stream of R's XDR serialisation: "X\\n", three int32 (format version 2, writer, min reader), then one item: a
REALSXP with attributes (flags 0x20e), int32 length, big-endian doubles, then its attribute pairlist: one LISTSXP node
(flags 0x402) tagged with the symbol "dim" (SYMSXP 1, CHARSXP "dim") holding an INTSXP of length 2, closed by NILVALUE
(0xfe).  make_rds_golden.py reads vectors without attributes; this file reads exactly this shape -- anything else raises.
"""
import gzip
import os
import struct
import sys

import numpy as np

REF = os.environ.get("BIGSNPR_REFERENCE", "/root/reference")


def read_rds_matrix(path):
    d = gzip.decompress(open(path, "rb").read())
    if d[:2] != b"X\n":
        raise ValueError("not an XDR serialisation: %r" % d[:2])
    version, _writer, _minreader = struct.unpack(">3i", d[2:14])
    if version != 2:
        raise ValueError("serialisation version %d not handled" % version)
    flags, length = struct.unpack(">2i", d[14:22])
    if flags & 0xFF != 14 or not flags & 0x200:
        raise ValueError("not a REALSXP with attributes (flags %#x)" % flags)
    vals = np.frombuffer(d, dtype=">f8", count=length, offset=22).astype(np.float64)
    o = 22 + 8 * length
    node, sym, chflags, chlen = struct.unpack(">4i", d[o:o + 16])
    if node != 0x402 or sym != 1 or chflags & 0xFF != 9:
        raise ValueError("attribute pairlist not handled")
    o += 16
    tag = d[o:o + chlen].decode()
    o += chlen
    iflags, ilen = struct.unpack(">2i", d[o:o + 8])
    if tag != "dim" or iflags & 0xFF != 13 or ilen != 2:
        raise ValueError("only a 'dim' attribute is handled")
    nrow, ncol = struct.unpack(">2i", d[o + 8:o + 16])
    o += 16
    if struct.unpack(">i", d[o:o + 4])[0] != 0xFE or o + 4 != len(d) or nrow * ncol != length:
        raise ValueError("trailing data")
    return vals.reshape((nrow, ncol), order="F")


def main():
    td = os.path.join(REF, "tests", "testthat", "testdata")
    scores = read_rds_matrix(os.path.join(td, "scores-PRS.rds"))
    thr = np.arange(11) * 0.5  # seq(0, 5, by = 0.5) of tests/testthat/test-6-PRS.R:34
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "prs_scores.npz")
    np.savez_compressed(out, scores=scores, thr=thr)
    print("wrote", out, "scores", scores.shape)


if __name__ == "__main__":
    sys.exit(main())
