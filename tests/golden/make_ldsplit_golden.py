"""Regenerates tests/golden/ldsplit.npz from the reference's own RDS fixtures of tests/testthat/test-4-split-LD.R (run
where a reference checkout exists, BIGSNPR_REFERENCE; the tests only read the committed .npz):

  tests/testthat/testdata/spMat.rds         401 x 401 dsCMatrix (slots p, i, x, Dim, uplo kept)
  tests/testthat/testdata/split_before.rds  tibble of snp_ldsplit before v1.10.1 (columns cost, n_block kept)

RDS = gzip stream of R's XDR serialisation: "X\n", three int32 (format version, writer, min reader), in version 3 the
native encoding's name, then one item.  _Reader parses the subset these two files use; anything else raises.
"""
import gzip
import os
import struct
import sys

import numpy as np

REF = os.environ.get("BIGSNPR_REFERENCE", "/root/reference")


class _Reader:
    """The subset of R's XDR serialisation (versions 2 and 3) that S4 objects and lists use: vectors, pairlists, symbols,
    CHARSXPs, S4 objects and their attributes (S4 slots are attributes), with back-references to symbols.  Returns plain
    Python values: numpy arrays, lists of str, dicts {"value": ..., "attributes": {...}}."""

    def __init__(self, d):
        self.d, self.o, self.refs = d, 0, []

    def i32(self):
        (v,) = struct.unpack_from(">i", self.d, self.o)
        self.o += 4
        return v

    def item(self):
        flags = self.i32()
        sxp, has_attr, has_tag = flags & 0xFF, bool(flags & 0x200), bool(flags & 0x400)
        if sxp == 254:  # R_NilValue
            return None
        if sxp == 255:  # REFSXP: the reference index is in the flags' upper bits (or follows when 0)
            idx = flags >> 8
            return self.refs[(idx if idx else self.i32()) - 1]
        if sxp == 1:  # SYMSXP: its CHARSXP follows
            name = self.item()
            self.refs.append(name)
            return name
        if sxp == 9:  # CHARSXP
            n = self.i32()
            if n == -1:
                return None
            s = self.d[self.o:self.o + n].decode("utf-8")
            self.o += n
            return s
        if sxp in (2, 25):  # LISTSXP (pairlist) or S4SXP: attributes, then (pairlist only) tag, car, cdr
            attrs = self.item() if has_attr else None
            if sxp == 25:
                return {"value": None, "attributes": attrs or {}}
            out = {}
            while True:
                tag = self.item() if has_tag else None
                out[tag] = self.item()
                nxt = self.i32()
                if nxt & 0xFF == 254:
                    return out
                has_tag = bool(nxt & 0x400)
                if nxt & 0xFF != 2 or nxt & 0x200:
                    raise ValueError("pairlist form not handled")
        n = self.i32()
        if sxp in (10, 13):  # LGLSXP, INTSXP
            v = np.frombuffer(self.d, dtype=">i4", count=n, offset=self.o).astype(np.int32)
            self.o += 4 * n
        elif sxp == 14:
            v = np.frombuffer(self.d, dtype=">f8", count=n, offset=self.o).astype(np.float64)
            self.o += 8 * n
        elif sxp == 16:  # STRSXP
            v = [self.item() for _ in range(n)]
        elif sxp == 19:  # VECSXP
            v = [self.item() for _ in range(n)]
        else:
            raise ValueError("SEXP type %d not handled" % sxp)
        return {"value": v, "attributes": self.item()} if has_attr else v


def read_rds(path):
    """Any RDS file within _Reader's subset."""
    d = gzip.decompress(open(path, "rb").read())
    if d[:2] != b"X\n":
        raise ValueError("not an XDR serialisation: %r" % d[:2])
    r = _Reader(d)
    r.o = 2
    version, _writer, _minreader = r.i32(), r.i32(), r.i32()
    if version == 3:
        r.o += r.i32()  # native encoding name
    elif version != 2:
        raise ValueError("serialisation version %d not handled" % version)
    out = r.item()
    if r.o != len(d):
        raise ValueError("trailing bytes")
    return out


def main():
    td = os.path.join(REF, "tests", "testthat", "testdata")
    # tests/testthat/test-4-split-LD.R:102,110: the 401-SNP dsCMatrix and the costs of snp_ldsplit before v1.10.1
    sp = read_rds(os.path.join(td, "spMat.rds"))["attributes"]
    before = read_rds(os.path.join(td, "split_before.rds"))
    cols = dict(zip(before["attributes"]["names"], before["value"]))
    out = os.path.join(os.path.dirname(os.path.abspath(__file__)), "ldsplit.npz")
    np.savez_compressed(out, p=sp["p"], i=sp["i"], x=sp["x"], Dim=sp["Dim"], uplo=np.array(sp["uplo"]),
                        before_cost=cols["cost"], before_n_block=cols["n_block"])
    print("wrote", out, "Dim", sp["Dim"], "uplo", sp["uplo"], "nnz", sp["x"].size, "before", cols["n_block"])


if __name__ == "__main__":
    sys.exit(main())
