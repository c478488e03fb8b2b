"""Host-side mirror of the reference's R interface for the packed-genotype hot path.

R is not available in the build image, so the host side above the C ABI (include/bsgpu.h) is Python,
mirroring the reference's operator interface: same function names, argument meaning (1-based
``ind_row`` / ``ind_col``, ``center`` / ``scale`` per selected column, ``ncores`` accepted and ignored)
and error behaviour, so the parity tests read like the reference's testthat files.  Reference:

    bed()/bed_light          R/bed-class.R:65-134,176-208      -> class Bed
    bed_prodVec / cprodVec   R/bed-mult-vec.R:58-75 / :20-37
    bed_counts / bed_MAF / bed_scaleBinom   R/binom-scaling.R:166-178 / :203-222 / :133-142
    obj.bed[i, j]            R/bed-mat-acc.R:21-38 (read_bed)
    bed_cor / snp_cor        R/corr.R:3-57,95-132
    bed_ld_scores / snp_ld_scores  R/ld-scores.R:3-72
    bed_tcrossprodSelf       R/bed-tcrossprodSelf.R:21-52
    bed_randomSVD            R/autoSVD.R:205-219
    bed_autoSVD              R/autoSVD.R:226-339 (control flow; outlier statistic pluggable, see the docstring)
    prod_and_rowSumsSq / bed_projectSelfPCA   src/bed-fun.cpp:103-133, R/bed-projectPCA.R:45-58,196-227
    multLinReg / bed_pcadapt / snp_pcadapt    src/multLinReg.cpp:8-88, R/pcadapt.R:3-27,61-81
    readbina2 / snp_readBed2, writebina / snp_writeBed   src/read-plink.cpp:61-80, src/write-plink.cpp:13-52
    as_SFBM / ld_scores_sfbm / snp_lassosum2   bigsparser's SFBM storage, src/ld-scores-sfbm.cpp:9-69, R/lassosum2.R:25-81
    snp_ldsplit / get_L / get_C   R/split-LD.R:3-40,99-138, src/split-LD.cpp:15-61,65-145,149-182
    sp_solve_sym / snp_ldpred2_inf   bigsparser's conjugate-gradient solve, R/LDpred2.R:27-42
    snp_ldpred2_auto / snp_ldpred2_grid   R/LDpred2.R:203-286, R/LDpred2.R:73-140 (seeded MRG32k3a streams, DESIGN.md §4.15, §4.18)
    snp_ldsc / snp_ldsc2   R/ldsc.R:1-224 (host NumPy; the LD scores of snp_ldsc2 come from ld_scores_sfbm)
    snp_PRS / snp_grid_PRS   R/PRS.R:36-76, R/SCT.R:201-246 (bsg_prs_grid: every keep set of a chromosome in one call)
    big_univLinReg           bigstatsr's univLinReg5 + R glue (not vendored; bsg_univlinreg), result class MHTest
    big_univLogReg           bigstatsr's IRLS + R glue (not vendored; bsg_univlogreg, glm.fit null model and refits here)
    big_spLinReg / big_spLogReg   bigstatsr's elastic net + CMSA (not vendored; bsg_splreg / bsg_splreg_dense, DESIGN.md §4.19)
    snp_grid_stacking        R/SCT.R:266-304 (big_spLinReg / big_spLogReg over snp_grid_PRS's scores, then the fold)

Everything computes on the GPU through libbsgpu; there is no CPU path here (LD score regression, a few
weighted least-squares fits on per-variant vectors, runs on the host).
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from . import _lib
from ._lib import BsgError, check, lib

ERROR_DIM = "Incompatibility between dimensions."
NA_INTEGER = -2147483648

LAYOUT_AUTO, LAYOUT_SNP_MAJOR, LAYOUT_SAMPLE_MAJOR = 0, 1, 2


def _i32(a):
    return np.ascontiguousarray(a, dtype=np.int32)


def _f64(a):
    return np.ascontiguousarray(a, dtype=np.float64)


def _pi(a):
    return None if a is None else a.ctypes.data_as(_lib.c_int_p)


def _pd(a):
    return None if a is None else a.ctypes.data_as(_lib.c_dbl_p)


def _count_lines(path):
    n = 0
    with open(path, "rb") as f:
        for _ in f:
            n += 1
    return n


class Bed:
    """A PLINK .bed staged in HBM: the ``bed`` RefClass of the reference (R/bed-class.R:65-134).

    ``Bed(bedfile)`` reads n from the .fam and m from the .bim like ``$nrow`` / ``$ncol`` do, validates
    the file exactly like ``bedXPtr`` (src/bed-acc-xptr.cpp:14-34) and stages the packed bytes once.
    ``col_range=(begin, end)`` (0-based, half open) stages only a column shard (multi-GPU).
    """

    def __init__(self, bedfile=None, nrow=None, ncol=None, device=0, layouts=LAYOUT_AUTO, col_range=None,
                 _handle=None, _shape=None):
        self._h = None
        self.bedfile = None
        if _handle is not None:
            self._h = _handle
            self.nrow, self.ncol = _shape
            self.bedfile = "<device>"
            return
        bedfile = os.path.expanduser(bedfile)
        self.bedfile = bedfile
        pre = bedfile[:-4] if bedfile.endswith(".bed") else bedfile
        for f in (bedfile, pre + ".bim", pre + ".fam"):
            if (nrow is None or ncol is None) and not os.path.exists(f):
                raise FileNotFoundError("File '%s' doesn't exist." % f)
        n = _count_lines(pre + ".fam") if nrow is None else int(nrow)
        m = _count_lines(pre + ".bim") if ncol is None else int(ncol)
        b, e = (0, m) if col_range is None else col_range
        h = C.c_void_p()
        check(lib().bsg_open_bed(bedfile.encode(), n, m, int(b), int(e), int(device), int(layouts), C.byref(h)))
        self._h = h
        self.nrow, self.ncol = n, int(e) - int(b)
        self.col_offset = int(b)

    # --- alternative constructors -----------------------------------------------------------
    @classmethod
    def from_packed(cls, packed, n, m, device=0, layouts=LAYOUT_AUTO):
        packed = np.ascontiguousarray(packed, dtype=np.uint8).reshape(-1)
        if packed.size != ((n + 3) // 4) * m:
            raise BsgError(5, "n or p does not match the dimensions of the file.")
        h = C.c_void_p()
        check(lib().bsg_open_packed(packed.ctypes.data_as(_lib.c_u8_p), int(n), int(m), int(device), int(layouts),
                                    C.byref(h)))
        return cls(_handle=h, _shape=(int(n), int(m)))

    @classmethod
    def synthetic(cls, n, m, seed=20250924, na_rate=0.0, col_offset=0, device=0, layouts=LAYOUT_AUTO, ld_rho=0.0,
                  ld_block=50):
        """Synthetic matrix generated on the device (SURVEY.md section 8d).  ld_rho > 0: haplotype blocks of `ld_block`
        SNPs whose alleles are copied from the previous SNP with probability ld_rho (correlated neighbours)."""
        h = C.c_void_p()
        if ld_rho > 0:
            check(lib().bsg_open_synth_ld(int(n), int(m), int(seed), float(na_rate), int(col_offset), float(ld_rho),
                                          int(ld_block), int(device), int(layouts), C.byref(h)))
        else:
            check(lib().bsg_open_synth(int(n), int(m), int(seed), float(na_rate), int(col_offset), int(device),
                                       int(layouts), C.byref(h)))
        return cls(_handle=h, _shape=(int(n), int(m)))

    @classmethod
    def from_fbm(cls, bytes_nm, code256=None, device=0, layouts=LAYOUT_AUTO):
        """FBM.code256 twin (snp_* functions): n x m raw bytes + the 256-entry code (default CODE_012)."""
        a = np.asfortranarray(bytes_nm, dtype=np.uint8)
        n, m = a.shape
        if code256 is None:
            code256 = np.full(256, np.nan)
            code256[:3] = [0, 1, 2]
        code256 = _f64(code256)
        h = C.c_void_p()
        check(lib().bsg_open_fbm256(a.ctypes.data_as(_lib.c_u8_p), n, m, _pd(code256), int(device), int(layouts),
                                    C.byref(h)))
        return cls(_handle=h, _shape=(n, m))

    # --- RefClass surface -------------------------------------------------------------------------
    @property
    def address(self):
        return self._h

    @property
    def light(self):
        return self

    @property
    def shape(self):
        return (self.nrow, self.ncol)

    def __len__(self):
        return self.nrow * self.ncol

    def __repr__(self):
        return "A 'bed' object with %d samples and %d variants." % (self.nrow, self.ncol)

    def rows_along(self):
        return np.arange(1, self.nrow + 1, dtype=np.int32)

    def cols_along(self):
        return np.arange(1, self.ncol + 1, dtype=np.int32)

    @property
    def map(self):
        """`$map` of the RefClass (R/bed-class.R:87-93): chromosome (str) and physical.pos read lazily from the .bim."""
        if getattr(self, "_map", None) is None:
            if not self.bedfile or self.bedfile.startswith("<"):
                raise ValueError("this handle has no .bim file: pass infos_chr / infos_pos")
            chrom, pos = [], []
            with open(self.bedfile[:-4] + ".bim") as f:
                for line in f:
                    p = line.split()
                    chrom.append(p[0])
                    pos.append(float(p[3]))
            off = getattr(self, "col_offset", 0)
            self._map = {"chromosome": np.array(chrom)[off:off + self.ncol],
                         "physical.pos": np.array(pos)[off:off + self.ncol]}
        return self._map

    @property
    def has_na(self):
        return bool(lib().bsg_has_na(self._h))

    @property
    def dosage_scale(self):
        """D when this handle holds dosages whose finite codes are multiples of 1 / D in 0..255 / D (CODE_DOSAGE: 100):
        such handles also serve bed_prodVec / bed_cprodVec and bed_randomSVD with an explicit fun_scaling.  0 otherwise."""
        return int(lib().bsg_dosage_scale(self._h))

    @property
    def layouts(self):
        return int(lib().bsg_layouts(self._h))

    @property
    def packed_bytes(self):
        return int(lib().bsg_packed_bytes(self._h))

    def export_packed(self):
        out = np.empty(((self.nrow + 3) // 4) * self.ncol, dtype=np.uint8)
        check(lib().bsg_export_packed(self._h, out.ctypes.data_as(_lib.c_u8_p)))
        return out

    def close(self):
        if self._h is not None:
            lib().bsg_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # obj.bed[i, j]  (R/bed-mat-acc.R:21-38; 1-based like R, NA -> NA_INTEGER)
    def __getitem__(self, key):
        i, j = key
        ind_row = self.rows_along() if i is None or (isinstance(i, slice) and i == slice(None)) else _i32(np.atleast_1d(i))
        ind_col = self.cols_along() if j is None or (isinstance(j, slice) and j == slice(None)) else _i32(np.atleast_1d(j))
        return read_bed(self, ind_row, ind_col)


class Group:
    """One matrix sharded by SNP columns over several GPUs driven by THIS process (bsg_group, SURVEY.md section 8e) -- the
    multi-GPU form an R session uses.  `ind_col` is global and 1-based like everywhere else; the library buckets it by
    owning device.  X.y ends in a sum over the devices done inside the epilogue kernel over NVLink peer memory."""

    def __init__(self, _handle):
        self._g = _handle
        L = lib()
        self.nrow, self.ncol, self.ndev = int(L.bsg_group_nrow(_handle)), int(L.bsg_group_ncol(_handle)), int(L.bsg_group_ndev(_handle))

    @classmethod
    def open(cls, bedfile, devices, nrow=None, ncol=None, layouts=LAYOUT_AUTO):
        bedfile = os.path.expanduser(bedfile)
        pre = bedfile[:-4] if bedfile.endswith(".bed") else bedfile
        n = _count_lines(pre + ".fam") if nrow is None else int(nrow)
        m = _count_lines(pre + ".bim") if ncol is None else int(ncol)
        dv = _i32(devices)
        g = C.c_void_p()
        check(lib().bsg_group_open_bed(bedfile.encode(), n, m, _pi(dv), dv.size, int(layouts), C.byref(g)))
        return cls(g)

    @classmethod
    def synthetic(cls, n, m, devices, seed=20250924, na_rate=0.0, ld_rho=0.0, ld_block=50, layouts=LAYOUT_AUTO):
        dv = _i32(devices)
        g = C.c_void_p()
        check(lib().bsg_group_open_synth(int(n), int(m), int(seed), float(na_rate), float(ld_rho), int(ld_block), _pi(dv),
                                         dv.size, int(layouts), C.byref(g)))
        return cls(g)

    def shard(self, i):
        """The per-device handle as a (non-owning) Bed plus its first global column (0-based)."""
        h = lib().bsg_group_shard(self._g, int(i))
        b0, b1 = lib().bsg_group_shard_begin(self._g, int(i)), lib().bsg_group_shard_begin(self._g, int(i) + 1)
        b = Bed(_handle=C.c_void_p(h), _shape=(self.nrow, b1 - b0))
        b.close = lambda: None  # owned by the group
        return b, b0

    def rows_along(self):
        return np.arange(1, self.nrow + 1, dtype=np.int32)

    def cols_along(self):
        return np.arange(1, self.ncol + 1, dtype=np.int32)

    def _args(self, ind_row, ind_col, center, scale):
        ir = None if ind_row is ... else _i32(ind_row)
        ic = None if ind_col is ... else _i32(ind_col)
        nr = self.nrow if ir is None else ir.size
        nc = self.ncol if ic is None else ic.size
        if (center is None) != (scale is None):
            raise ValueError("center and scale must be given together")
        if center is not None:
            center, scale = _f64(center), _f64(scale)
            if center.size != nc or scale.size != nc:
                raise ValueError(ERROR_DIM)
        return ir, nr, ic, nc, center, scale

    def prodVec(self, y_col, ind_row=..., ind_col=..., center=None, scale=None):
        ir, nr, ic, nc, center, scale = self._args(ind_row, ind_col, center, scale)
        y_col = _f64(y_col)
        if y_col.size != nc:
            raise ValueError(ERROR_DIM)
        out = np.empty(nr)
        check(lib().bsg_group_prodvec(self._g, _pi(ir), nr, _pi(ic), nc, _pd(center), _pd(scale), _pd(y_col), _pd(out)))
        return out

    def cprodVec(self, y_row, ind_row=..., ind_col=..., center=None, scale=None):
        ir, nr, ic, nc, center, scale = self._args(ind_row, ind_col, center, scale)
        y_row = _f64(y_row)
        if y_row.size != nr:
            raise ValueError(ERROR_DIM)
        out = np.empty(nc)
        check(lib().bsg_group_cprodvec(self._g, _pi(ir), nr, _pi(ic), nc, _pd(center), _pd(scale), _pd(y_row), _pd(out)))
        return out

    def randomSVD(self, ind_row=..., ind_col=..., center=None, scale=None, k=10, tol=1e-4, maxit=1000):
        """bed_randomSVD (binomial scaling computed per shard when center / scale are not given)."""
        ir, nr, ic, nc, center, scale = self._args(ind_row, ind_col, center, scale)
        d, u, v = np.empty(k), np.empty((k, nr)), np.empty((k, nc))
        c_out, s_out = np.empty(nc), np.empty(nc)
        niter, nops = C.c_int(0), C.c_int(0)
        check(lib().bsg_group_randomsvd(self._g, _pi(ir), nr, _pi(ic), nc, _pd(center), _pd(scale), int(k), float(tol),
                                        int(maxit), _pd(d), _pd(u), _pd(v), _pd(c_out), _pd(s_out), C.byref(niter),
                                        C.byref(nops)))
        return {"d": d, "u": u.T, "v": v.T, "niter": niter.value, "nops": nops.value, "center": c_out, "scale": s_out}

    def tcrossprodSelf(self, center, scale, ind_row=..., ind_col=...):
        ir, nr, ic, nc, center, scale = self._args(ind_row, ind_col, center, scale)
        K = np.empty((nr, nr))
        check(lib().bsg_group_tcrossprod(self._g, _pi(ir), nr, _pi(ic), nc, _pd(center), _pd(scale), _pd(K)))
        return K

    def scaleBinom(self, ind_row=...):
        """bed_scaleBinom over all columns: per-shard statistics concatenated (a gather, SURVEY.md section 8e)."""
        cs, ss = [], []
        for i in range(self.ndev):
            b, _ = self.shard(i)
            sc = bed_scaleBinom(b, ind_row)
            cs.append(sc["center"])
            ss.append(sc["scale"])
        return {"center": np.concatenate(cs), "scale": np.concatenate(ss)}

    def close(self):
        if self._g is not None:
            lib().bsg_group_close(self._g)
            self._g = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bed(bedfile, **kw):
    """Wrapper constructor (R/bed-class.R:146)."""
    return Bed(bedfile, **kw)


def _assert_bed(obj):
    if not isinstance(obj, Bed):
        raise TypeError("'obj.bed' is not of class 'bed' or 'bed_light'.")


def _ind(obj, ind_row, ind_col):
    if ind_row is None:
        raise ValueError("'ind.row' can't be `NULL`.")
    if ind_col is None:
        raise ValueError("'ind.col' can't be `NULL`.")
    return _i32(ind_row), _i32(ind_col)


def _dflt(obj, ind_row, ind_col):
    return (obj.rows_along() if ind_row is ... else ind_row), (obj.cols_along() if ind_col is ... else ind_col)


def _assert_lengths(a, b):
    if len(a) != len(b):
        raise ValueError(ERROR_DIM)


class View:
    """Device-resident accessor state (ind.row, ind.col, center, scale): bsg_view."""

    def __init__(self, obj, ind_row=..., ind_col=..., center=None, scale=None):
        _assert_bed(obj)
        ind_row, ind_col = _dflt(obj, ind_row, ind_col)
        ind_row, ind_col = _ind(obj, ind_row, ind_col)
        self.obj = obj
        self.nr, self.nc = ind_row.size, ind_col.size
        if (center is None) != (scale is None):
            raise ValueError("center and scale must be given together")
        if center is not None:
            center, scale = _f64(center), _f64(scale)
            _assert_lengths(center, ind_col)
            _assert_lengths(scale, ind_col)
        v = C.c_void_p()
        check(lib().bsg_view_create(obj._h, _pi(ind_row), self.nr, _pi(ind_col), self.nc, _pd(center), _pd(scale),
                                    C.byref(v)))
        self._v = v

    def prodvec(self, y_col):
        y_col = _f64(y_col)
        if y_col.size != self.nc:
            raise ValueError(ERROR_DIM)
        out = np.empty(self.nr)
        check(lib().bsg_view_prodvec(self._v, _pd(y_col), _pd(out)))
        return out

    def cprodvec(self, y_row):
        y_row = _f64(y_row)
        if y_row.size != self.nr:
            raise ValueError(ERROR_DIM)
        out = np.empty(self.nc)
        check(lib().bsg_view_cprodvec(self._v, _pd(y_row), _pd(out)))
        return out

    def prodvec_dev(self, x_ptr, out_ptr, stream=0):
        check(lib().bsg_view_prodvec_dev(self._v, int(x_ptr), int(out_ptr), int(stream) or None))

    def cprodvec_dev(self, x_ptr, out_ptr, stream=0):
        check(lib().bsg_view_cprodvec_dev(self._v, int(x_ptr), int(out_ptr), int(stream) or None))

    def close(self):
        if self._v is not None:
            lib().bsg_view_destroy(self._v)
            self._v = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


def bed_prodVec(obj_bed, y_col, ind_row=..., ind_col=..., center=None, scale=None, ncores=1):
    """Product between a "bed" object and a vector (R/bed-mult-vec.R:58-75)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    y_col = _f64(y_col)
    _assert_lengths(y_col, ind_col)
    center = np.zeros(ind_col.size) if center is None else _f64(center)
    _assert_lengths(center, ind_col)
    scale = np.ones(ind_col.size) if scale is None else _f64(scale)
    _assert_lengths(scale, ind_col)
    out = np.empty(ind_row.size)
    check(lib().bsg_prodvec(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                            _pd(scale), _pd(y_col), _pd(out)))
    return out


def bed_cprodVec(obj_bed, y_row, ind_row=..., ind_col=..., center=None, scale=None, ncores=1):
    """Cross-product between a "bed" object and a vector (R/bed-mult-vec.R:20-37)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    y_row = _f64(y_row)
    _assert_lengths(y_row, ind_row)
    center = np.zeros(ind_col.size) if center is None else _f64(center)
    _assert_lengths(center, ind_col)
    scale = np.ones(ind_col.size) if scale is None else _f64(scale)
    _assert_lengths(scale, ind_col)
    out = np.empty(ind_col.size)
    check(lib().bsg_cprodvec(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                             _pd(scale), _pd(y_row), _pd(out)))
    return out


def bed_colstats(obj_bed, ind_row=..., ind_col=..., ncores=1):
    """src/bed-fun.cpp:9-46 -> dict(sumX, denoX, nb_nona_col); warns like the reference (:40-41)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    m = ind_col.size
    sumX, denoX, nb = np.empty(m), np.empty(m), np.empty(m, dtype=np.int32)
    n_bad = C.c_int(0)
    check(lib().bsg_colstats(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), m, _pd(sumX), _pd(denoX), _pi(nb),
                             C.byref(n_bad)))
    if n_bad.value > 0:
        import warnings

        warnings.warn("%d variants have >50%% missing values." % n_bad.value)
    return {"sumX": sumX, "denoX": denoX, "nb_nona_col": nb}


def bed_scaleBinom(obj_bed, ind_row=..., ind_col=..., ncores=1):
    """Binomial(2, p) scaling (R/binom-scaling.R:133-142)."""
    st = bed_colstats(obj_bed, ind_row, ind_col, ncores)
    with np.errstate(all="ignore"):
        af = st["sumX"] / (2 * st["nb_nona_col"])
        return {"center": 2 * af, "scale": np.sqrt(2 * af * (1 - af))}


def bed_counts(obj_bed, ind_row=..., ind_col=..., byrow=False, ncores=1):
    """Counts of 0s, 1s, 2s and NAs by variant (or by individual): R/binom-scaling.R:166-178 -> (4, k)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    k = ind_row.size if byrow else ind_col.size
    res = np.zeros((k, 4), dtype=np.int32)
    f = lib().bsg_row_counts if byrow else lib().bsg_col_counts
    check(f(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pi(res)))
    return res.T


def bed_MAF(obj_bed, ind_row=..., ind_col=..., ncores=1):
    """Allele frequencies (R/binom-scaling.R:203-222)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    counts = bed_counts(obj_bed, ind_row, ind_col, False, ncores).astype(np.int64)
    ac = counts[1] + 2 * counts[2]
    nb_nona = ind_row.size - counts[3]
    with np.errstate(all="ignore"):
        af = ac / (2 * nb_nona)
    return {"ac": ac, "mac": np.minimum(ac, 2 * nb_nona - ac), "af": af, "maf": np.minimum(af, 1 - af), "N": nb_nona}


def snp_colstats(G, ind_row=..., ind_col=..., ncores=1):
    """src/colstats.cpp:8-35 on an FBM-backed handle."""
    ind_row, ind_col = _ind(G, *_dflt(G, ind_row, ind_col))
    m = ind_col.size
    sumX, denoX = np.empty(m), np.empty(m)
    check(lib().bsg_snp_colstats(G._h, _pi(ind_row), ind_row.size, _pi(ind_col), m, _pd(sumX), _pd(denoX)))
    return {"sumX": sumX, "denoX": denoX}


def code256_dosage_scale(code256):
    """The smallest integer D in 1..255 such that D * v is an integer in 0..255 for every finite value v of the FBM.code256
    table (and every other value is NA), else 0 (see include/bsgpu.h)."""
    code256 = _f64(code256)
    if code256.size != 256:
        raise ValueError("code256 must have 256 values.")
    return int(lib().bsg_code256_dosage_scale(_pd(code256)))


def snp_scaleBinom(nploidy=2):
    """R/binom-scaling.R:62-77: returns the scaling function."""

    def f(X, ind_row=..., ind_col=..., ncores=1):
        ind_row2, _ = _dflt(X, ind_row, ind_col)
        af = snp_colstats(X, ind_row, ind_col, ncores)["sumX"] / (len(ind_row2) * nploidy)
        with np.errstate(all="ignore"):
            return {"center": nploidy * af, "scale": np.sqrt(nploidy * af * (1 - af))}

    return f


def snp_MAF(G, ind_row=..., ind_col=..., nploidy=2, ncores=1):
    """R/binom-scaling.R:94-106."""
    ind_row2, _ = _dflt(G, ind_row, ind_col)
    af = snp_colstats(G, ind_row, ind_col, ncores)["sumX"] / (len(ind_row2) * nploidy)
    return np.minimum(af, 1 - af)


def read_bed(obj_bed, ind_row, ind_col, na_val=NA_INTEGER):
    """src/bed-mat-acc.cpp:8-26 -> int32 (nr, nc)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    res = np.empty((ind_col.size, ind_row.size), dtype=np.int32)
    check(lib().bsg_read_bed(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, int(na_val), _pi(res)))
    return res.T


def read_bed_scaled(obj_bed, ind_row, ind_col, center, scale):
    """src/bed-mat-acc.cpp:30-49 -> float64 (nr, nc)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    center, scale = _f64(center), _f64(scale)
    if center.size != ind_col.size or scale.size != ind_col.size:
        raise ValueError(ERROR_DIM)
    res = np.empty((ind_col.size, ind_row.size), dtype=np.float64)
    check(lib().bsg_read_bed_scaled(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                                    _pd(scale), _pd(res)))
    return res.T


def cor_thresholds(n_row, alpha=1.0, thr_r2=0.0):
    """R/corr.R:17-23,29: THR = q / sqrt(k - 2 + q^2) with q = qt(alpha/2, k-2, upper); pmax with sqrt(thr_r2)."""
    from scipy import stats

    k = np.arange(1, n_row + 1, dtype=np.float64)
    with np.errstate(all="ignore"):
        q = stats.t.isf(alpha / 2, df=k - 2)
        thr = q / np.sqrt(k - 2 + q * q)
        return np.where(np.isnan(thr), np.nan, np.maximum(thr, np.sqrt(thr_r2)))


def corMat(obj, rowInd, colInd, size, thr, pos, fill_diag=True, ncores=1):
    """src/corr.cpp:102-126 -> CSC pieces (p, i, x); i 0-based ascending, diagonal last."""
    rowInd, colInd = _i32(rowInd), _i32(colInd)
    thr, pos = _f64(thr), _f64(pos)
    if pos.size != colInd.size:
        raise ValueError(ERROR_DIM)
    if thr.size != rowInd.size:
        raise ValueError(ERROR_DIM)
    p = np.zeros(colInd.size + 1, dtype=np.int64)
    pi, px = _lib.c_int_p(), _lib.c_dbl_p()
    check(lib().bsg_cor(obj._h, _pi(rowInd), rowInd.size, _pi(colInd), colInd.size, float(size), _pd(thr), _pd(pos),
                        int(bool(fill_diag)), p.ctypes.data_as(_lib.c_i64_p), C.byref(pi), C.byref(px)))
    nnz = int(p[-1])
    return p, _adopt(pi, C.c_int32, np.int32, nnz), _adopt(px, C.c_double, np.float64, nnz)


class _CBuffer:
    """Owner of an array the library allocated: released with bsg_free when the last numpy view is gone."""

    def __init__(self, ptr):
        self._ptr = ptr

    def __del__(self):
        try:
            lib().bsg_free(self._ptr)
        except Exception:  # interpreter shutdown
            pass


def _adopt(ptr, ctype, dtype, count):
    """numpy array over a library-owned buffer WITHOUT a copy (configs[2]'s CSC arrays are 1.2 GB: a copy doubles the
    host time of the call); the buffer lives as long as the array or any view of it."""
    owner = _CBuffer(C.cast(ptr, C.c_void_p))
    if count <= 0:
        return np.zeros(0, dtype=dtype)
    buf = (ctype * count).from_address(C.addressof(ptr.contents))
    buf._owner = owner
    return np.frombuffer(buf, dtype=dtype, count=count)


def _cor0(obj, ind_row, ind_col, size, alpha, thr_r2, fill_diag, infos_pos, ncores):
    ind_row, ind_col = _ind(obj, *_dflt(obj, ind_row, ind_col))
    if infos_pos is None:
        infos_pos = 1000.0 * np.arange(1, ind_col.size + 1)
    infos_pos = _f64(infos_pos)
    _assert_lengths(infos_pos, ind_col)
    if np.any(np.diff(infos_pos) < 0):
        raise ValueError("'infos.pos' is not sorted.")
    thr = cor_thresholds(ind_row.size, alpha, thr_r2)
    p, i, x = corMat(obj, ind_row, ind_col, size * 1000.0, thr, infos_pos, fill_diag, ncores)
    if np.isnan(x).any():
        import warnings

        warnings.warn("NA or NaN values in the resulting correlation matrix.")
    return p, i, x


def bed_cor(obj_bed, ind_row=..., ind_col=..., size=500, alpha=1.0, thr_r2=0.0, fill_diag=True, infos_pos=None, ncores=1):
    """Correlation matrix (R/corr.R:116-132): CSC (p, i, x) of the upper-triangular dsCMatrix."""
    _assert_bed(obj_bed)
    return _cor0(obj_bed, ind_row, ind_col, size, alpha, thr_r2, fill_diag, infos_pos, ncores)


snp_cor = bed_cor  # R/corr.R:95-110 (FBM-backed handles share the packed kernels)


def bed_ld_scores(obj_bed, ind_row=..., ind_col=..., size=500, infos_pos=None, ncores=1):
    """LD scores (R/ld-scores.R:59-72)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    if infos_pos is None:
        infos_pos = 1000.0 * np.arange(1, ind_col.size + 1)
    infos_pos = _f64(infos_pos)
    _assert_lengths(infos_pos, ind_col)
    if np.any(np.diff(infos_pos) < 0):
        raise ValueError("'infos.pos' is not sorted.")
    out = np.empty(ind_col.size)
    check(lib().bsg_ld_scores(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, float(size) * 1000.0,
                              _pd(infos_pos), _pd(out)))
    return out


snp_ld_scores = bed_ld_scores


def bed_tcrossprodSelf(obj_bed, fun_scaling=bed_scaleBinom, ind_row=..., ind_col=..., block_size=None):
    """tcrossprod / GRM (R/bed-tcrossprodSelf.R:21-52).  The R block loop is one C-ABI call; ``block_size``
    is accepted for signature compatibility.  Returns (K, center, scale)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    ms = fun_scaling(obj_bed, ind_row=ind_row, ind_col=ind_col)
    center, scale = _f64(ms["center"]), _f64(ms["scale"])
    n = ind_row.size
    K = np.empty((n, n))
    check(lib().bsg_tcrossprod(obj_bed._h, _pi(ind_row), n, _pi(ind_col), ind_col.size, _pd(center), _pd(scale), _pd(K)))
    return K, center, scale


def bed_randomSVD(obj_bed, fun_scaling=bed_scaleBinom, ind_row=..., ind_col=..., k=10, tol=1e-4, verbose=False,
                  ncores=1, maxit=1000):
    """Randomized partial SVD (R/autoSVD.R:205-219) -> dict(d, u, v, niter, nops, center, scale)."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    n, m = ind_row.size, ind_col.size
    center = scale = None
    if fun_scaling is not bed_scaleBinom:
        ms = fun_scaling(obj_bed, ind_row=ind_row, ind_col=ind_col)
        center, scale = _f64(ms["center"]), _f64(ms["scale"])
    d = np.empty(k)
    u = np.empty((k, n))
    v = np.empty((k, m))
    c_out, s_out = np.empty(m), np.empty(m)
    niter, nops = C.c_int(0), C.c_int(0)
    check(lib().bsg_randomsvd(obj_bed._h, _pi(ind_row), n, _pi(ind_col), m, _pd(center), _pd(scale), int(k), float(tol),
                              int(maxit), _pd(d), _pd(u), _pd(v), _pd(c_out), _pd(s_out), C.byref(niter), C.byref(nops)))
    nconv = int(lib().bsg_randomsvd_nconv())
    if 0 <= nconv < k:  # RSpectra::svds behind big_randomSVD: "only %d singular values converged"
        import warnings

        warnings.warn("only %d singular values converged after %d restarts (maxit = %d)." % (nconv, niter.value, maxit))
    return {"d": d, "u": u.T, "v": v.T, "niter": niter.value, "nops": nops.value, "center": c_out, "scale": s_out}


def _get_intervals(x, n=2):
    """R/autoSVD.R:4-12: regroup consecutive integers (runs of at least n) into [start, stop] rows."""
    x = np.asarray(x, dtype=np.int64)
    out, i = [], 0
    while i < x.size:
        j = i
        while j + 1 < x.size and x[j + 1] - x[j] == 1:
            j += 1
        if j - i + 1 >= max(n, 2):  # rle(diff(x)): a run needs at least one unit step, singletons never count
            out.append((int(x[i]), int(x[j])))
        i = j + 1
    return out


def _outlier_callable(outlier_fun, roll_size, alpha_tukey):
    """"default": the reference's detector (OGK distance -> rolling mean -> adjusted Tukey fence, outliers.py);
    None: never flag a variant (the loop stops after the first SVD); a callable is used as is."""
    if outlier_fun == "default":
        from .outliers import autosvd_outlier_fun

        return autosvd_outlier_fun(roll_size, alpha_tukey)
    return outlier_fun


def snp_autoSVD(G, infos_chr, infos_pos=None, ind_row=..., ind_col=..., fun_scaling=None, thr_r2=0.2, size=None, k=10,
                roll_size=50, int_min_size=20, alpha_tukey=0.05, min_mac=10, min_maf=0.02, max_iter=5, ncores=1,
                verbose=False, outlier_fun="default"):
    """R/autoSVD.R:67-186: the FBM.code256 twin of bed_autoSVD (snp_MAF -> snp_clumping -> randomSVD loop); `G` is a
    handle staged from an FBM (Bed.from_fbm).  Same remark on the outlier statistic as bed_autoSVD."""
    outlier_fun = _outlier_callable(outlier_fun, roll_size, alpha_tukey)
    infos_chr = np.asarray(infos_chr)
    _assert_lengths(infos_chr, G.cols_along())
    if infos_pos is not None:
        _assert_lengths(infos_pos, infos_chr)
    return _auto_svd(G, infos_chr, None if infos_pos is None else _f64(infos_pos), ind_row, ind_col,
                     fun_scaling or snp_scaleBinom(), thr_r2, size, k, int_min_size, min_mac, min_maf, max_iter, ncores,
                     verbose, outlier_fun, fbm=True)


def bed_autoSVD(obj_bed, ind_row=..., ind_col=..., fun_scaling=bed_scaleBinom, thr_r2=0.2, size=None, k=10,
                roll_size=50, int_min_size=20, alpha_tukey=0.05, min_mac=10, min_maf=0.02, max_iter=5, ncores=1,
                verbose=False, outlier_fun="default"):
    """Truncated SVD while limiting LD (R/autoSVD.R:226-339): MAC / MAF filter (bed_MAF) -> clumping on MAC
    (bed_clumping) -> bed_randomSVD, then up to `max_iter` rounds of outlier-variant removal, same arguments and defaults
    as the reference (roll.size = 50, int.min.size = 20, alpha.tukey = 0.05).

    The engine steps (counts, clumping, SVD) run on the GPU.  The outlier statistic (R/autoSVD.R:295-302) is host-side
    code on the (m x k) loadings: the default restates bigutilsr's dist_ogk / rollmean / tukey_mc_up from their published
    algorithms (bigsnpr_b200/outliers.py -- bigutilsr is un-vendored, so this step's numbers are NOT pinned against the
    reference; every engine step is).  ``outlier_fun`` may also be a callable ``(v, infos_chr_keep) -> 0-based indices
    into the kept variants`` or None (no pruning).  Returns the SVD dict plus ``subset`` (1-based kept columns) and
    ``lrldr`` (list of (chr, start, stop, iter))."""
    _assert_bed(obj_bed)
    outlier_fun = _outlier_callable(outlier_fun, roll_size, alpha_tukey)
    return _auto_svd(obj_bed, obj_bed.map["chromosome"], obj_bed.map["physical.pos"], ind_row, ind_col, fun_scaling, thr_r2,
                     size, k, int_min_size, min_mac, min_maf, max_iter, ncores, verbose, outlier_fun, fbm=False)


def _auto_svd(obj_bed, infos_chr, infos_pos, ind_row, ind_col, fun_scaling, thr_r2, size, k, int_min_size, min_mac, min_maf,
              max_iter, ncores, verbose, outlier_fun, fbm):
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    if size is None and thr_r2 is not None and not np.isnan(thr_r2):
        size = 100 / thr_r2
    say = print if verbose else (lambda *a, **k: None)
    if not (min_mac > 0 and min_maf > 0):
        raise ValueError("You cannot use variants with no variation; set min.mac > 0 and min.maf > 0.")
    if fbm and obj_bed.dosage_scale:
        # dosages have no hard-call counts: R/autoSVD.R:96-101, snp_MAF and maf < max(min.maf, min.mac / (2 n))
        maf = snp_MAF(obj_bed, ind_row, ind_col, ncores=ncores)
        nok = maf < max(min_maf, min_mac / (2 * ind_row.size))
    else:
        info = bed_MAF(obj_bed, ind_row, ind_col, ncores)
        nok = (info["mac"] < min_mac) | (info["maf"] < min_maf)
    say("Discarding %d variant%s with MAC < %s or MAF < %s." % (nok.sum(), "s" if nok.sum() > 1 else "", min_mac, min_maf))
    ind_keep = ind_col[~nok]
    if thr_r2 is None or np.isnan(thr_r2):
        say("Skipping clumping.")
    else:
        excl = np.setdiff1d(obj_bed.cols_along(), ind_keep)
        if fbm:
            ind_keep = snp_clumping(obj_bed, infos_chr, ind_row=ind_row, exclude=excl, thr_r2=thr_r2, size=size,
                                    infos_pos=infos_pos, ncores=ncores)
        else:
            ind_keep = bed_clumping(obj_bed, ind_row=ind_row, exclude=excl, thr_r2=thr_r2, size=size, ncores=ncores,
                                    infos_chr=infos_chr, infos_pos=infos_pos)
        say("Phase of clumping (on MAC) at r^2 > %s.. keep %d variants." % (thr_r2, ind_keep.size))
    it, lrldr = 0, []
    while True:
        it += 1
        svd = bed_randomSVD(obj_bed, fun_scaling=fun_scaling, ind_row=ind_row, ind_col=ind_keep, k=k, ncores=ncores)
        if it > max_iter:
            say("Maximum number of iterations reached.")
            break
        excl = np.zeros(0, dtype=np.int64) if outlier_fun is None else np.asarray(
            outlier_fun(svd["v"], infos_chr[ind_keep - 1]), dtype=np.int64)
        say("%d outlier variant%s detected.." % (excl.size, "s" if excl.size > 1 else ""))
        if excl.size == 0:
            say("Converged!")
            break
        for a, b in _get_intervals(np.sort(excl) + 1, n=int_min_size):
            seq = np.arange(a, b + 1) - 1
            chrs = infos_chr[ind_keep[seq] - 1]
            vals, cnts = np.unique(chrs, return_counts=True)
            ch = vals[np.argmax(cnts)]
            in_chr = chrs == ch
            if infos_pos is not None:
                rng_pos = infos_pos[ind_keep[seq[in_chr]] - 1]
                lrldr.append((ch, float(rng_pos.min()), float(rng_pos.max()), it))
        ind_keep = np.delete(ind_keep, excl)
    svd = dict(svd)
    svd["subset"] = ind_keep
    svd["lrldr"] = sorted(lrldr)
    return svd


def clumping_chr(G, rowInd, colInd, ordInd, rankInd, pos, sumX, denoX, size, thr, ncores=1):
    """src/clumping.cpp:10-91 (FBM.code256 handle) -> keep (int32 0/1 per column of colInd)."""
    rowInd, colInd, ordInd = _i32(rowInd), _i32(colInd), _i32(ordInd)
    pos, sumX, denoX = _f64(pos), _f64(sumX), _f64(denoX)
    for v in (pos, sumX, denoX, ordInd):
        if v.size != colInd.size:
            raise ValueError(ERROR_DIM)
    keep = np.full(colInd.size, -1, dtype=np.int32)
    check(lib().bsg_clumping_chr_fbm(G._h, _pi(rowInd), rowInd.size, _pi(colInd), colInd.size, _pd(sumX), _pd(denoX),
                                     _pi(ordInd), _pd(pos), float(size), float(thr), _pi(keep)))
    return keep


def snp_clumping(G, infos_chr, ind_row=..., S=None, thr_r2=0.2, size=None, infos_pos=None, exclude=None, ncores=1):
    """LD clumping on an FBM.code256 handle (R/clumping.R:62-137): sorted 1-based indices of the variants kept."""
    _assert_bed(G)
    infos_chr = np.asarray(infos_chr)
    _assert_lengths(infos_chr, G.cols_along())
    if infos_pos is not None:
        _assert_lengths(infos_pos, infos_chr)
    if S is not None:
        _assert_lengths(S, infos_chr)
    ind_row = G.rows_along() if ind_row is ... else _i32(ind_row)
    if size is None:
        size = 100 / thr_r2
    m = G.ncol
    noexcl = np.setdiff1d(np.arange(1, m + 1), np.asarray([] if exclude is None else exclude, dtype=np.int64))
    kept = []
    for chrom in sorted(set(infos_chr[noexcl - 1].tolist())):
        ind_chr = noexcl[infos_chr[noexcl - 1] == chrom].astype(np.int32)
        st = snp_colstats(G, ind_row, ind_chr, ncores)
        n = ind_row.size
        if S is None:
            af = st["sumX"] / (2 * n)
            S_chr = np.minimum(af, 1 - af)
        else:
            S_chr = np.asarray(S)[ind_chr - 1]
        ordv = (np.argsort(-np.asarray(S_chr, dtype=np.float64), kind="stable") + 1).astype(np.int32)
        if infos_pos is None:
            pos_chr, sz = np.arange(1, ind_chr.size + 1, dtype=np.float64), float(size)
        else:
            pos_chr, sz = _f64(np.asarray(infos_pos)[ind_chr - 1]), size * 1000.0
            if np.any(np.diff(pos_chr) < 0):
                raise ValueError("'pos.chr' is not sorted.")
        keep = clumping_chr(G, ind_row, ind_chr, ordv, None, pos_chr, st["sumX"], st["denoX"], sz, thr_r2, ncores)
        if not np.all((keep == 0) | (keep == 1)):
            raise RuntimeError("clumping left undecided variants")
        kept.append(ind_chr[keep == 1])
    return np.sort(np.concatenate(kept)) if kept else np.zeros(0, dtype=np.int32)


def clumping_chr_cached(G, keep, sqcor, spInd, rowInd, colInd, ordInd, rankInd, pos, sumX, denoX, size, thr, ncores=1):
    """src/clumping-cached.cpp:11-110: writes 0 / 1 into `keep` (int32, one per column of colInd) and returns `sqcor` as
    passed.  The reference's r2 cache never changes a decision, so the call is clumping_chr's (bsg_clumping_chr_fbm)."""
    if np.asarray(spInd).size != np.asarray(colInd).size:
        raise ValueError(ERROR_DIM)
    keep[:] = clumping_chr(G, rowInd, colInd, ordInd, rankInd, pos, sumX, denoX, size, thr, ncores)
    return sqcor


class GridClumping(list):
    """snp_grid_clumping's result: one list per chromosome of 1-based index arrays, with the `grid` attribute (dict of
    columns size, thr_r2, grp_num, thr_imp, one row per keep set of a chromosome)."""

    grid = None


def _order_decreasing(x):
    """R's order(x, decreasing = TRUE): ties by position, NA last."""
    x = np.asarray(x, dtype=np.float64)
    key = np.where(np.isnan(x), np.inf, -x)
    return np.argsort(key, kind="stable")


def snp_grid_clumping(G, infos_chr, infos_pos, lpS, ind_row=..., grid_thr_r2=(0.01, 0.05, 0.1, 0.2, 0.5, 0.8, 0.95),
                      grid_base_size=(50, 100, 200, 500), infos_imp=None, grid_thr_imp=1, groups=None, exclude=None,
                      ncores=1):
    """Grid of clumping (R/SCT.R:32-151) on an FBM.code256 handle: for every chromosome, every (thr_imp, group) subset and
    every (thr_r2, base_size) point, the indices kept by clumping_chr with size 1000 * base_size / thr_r2 bp.  One
    bsg_grid_clumping_chr call per chromosome computes each pair's statistic once and resolves every instance together."""
    _assert_bed(G)
    cols = G.cols_along()
    infos_chr = np.asarray(infos_chr)
    infos_imp = np.ones(cols.size) if infos_imp is None else _f64(infos_imp)
    for v in (infos_chr, infos_pos, infos_imp, lpS):
        _assert_lengths(v, cols)
    infos_pos, lpS = _f64(infos_pos), _f64(lpS)
    if groups is None:
        groups = [cols]
    if not isinstance(groups, (list, tuple)):
        raise TypeError("'groups' is not of class 'list'.")
    groups = [np.asarray(gr, dtype=np.int64).reshape(-1) for gr in groups]
    ind_row = G.rows_along() if ind_row is ... else _i32(ind_row)
    THR_IMP = np.unique(np.asarray(grid_thr_imp, dtype=np.float64).reshape(-1))
    THR_CLMP = np.unique(np.asarray(grid_thr_r2, dtype=np.float64).reshape(-1))
    BASE = np.unique(np.asarray(grid_base_size, dtype=np.float64).reshape(-1))
    # expand.grid(size, thr.r2, grp.num, thr.imp): the first factor varies fastest
    g_imp, g_grp, g_thr, g_size = (a.ravel() for a in np.meshgrid(THR_IMP, np.arange(1, len(groups) + 1), THR_CLMP, BASE,
                                                                   indexing="ij"))
    grid = {"size": np.trunc(g_size / g_thr).astype(np.int32), "thr_r2": g_thr, "grp_num": g_grp.astype(np.int32),
            "thr_imp": g_imp}
    # the points of one subset, in the order of the reference's loops (thr.r2 outer, base.size inner)
    p_thr, p_base = (a.ravel() for a in np.meshgrid(THR_CLMP, BASE, indexing="ij"))
    p_size = 1000 * p_base / p_thr  # R/SCT.R:133, in bp
    npt = p_thr.size
    excl = np.asarray([] if exclude is None else exclude, dtype=np.int64)
    noexcl = np.arange(1, infos_chr.size + 1)
    noexcl = noexcl[~np.isin(noexcl, excl)]
    out = GridClumping()
    for chrom in sorted(set(infos_chr[noexcl - 1].tolist())):
        ind_chr = noexcl[infos_chr[noexcl - 1] == chrom].astype(np.int32)
        pos_chr = infos_pos[ind_chr - 1]
        st = snp_colstats(G, ind_row, ind_chr, ncores)
        if np.any(np.diff(pos_chr) < 0):
            raise ValueError("'pos.chr' is not sorted.")
        info_chr, S_chr = infos_imp[ind_chr - 1], lpS[ind_chr - 1]
        cur = np.arange(ind_chr.size)  # positions within ind_chr that pass the thresholds of imputation so far
        sub_cols, sub_ords = [], []
        for thr_imp in THR_IMP:
            cur = cur[info_chr[cur] >= thr_imp]
            for group in groups:
                sub = cur[np.isin(ind_chr[cur], group)]
                sub_cols.append(sub)
                sub_ords.append(_order_decreasing(S_chr[sub]))
        lens = _i32([s.size for s in sub_cols])
        cat = lambda parts: _i32(np.concatenate(parts) + 1) if parts else np.zeros(0, dtype=np.int32)  # noqa: E731
        keep = np.full(max(int(lens.sum()) * npt, 1), -1, dtype=np.int32)
        check(lib().bsg_grid_clumping_chr(G._h, _pi(ind_row), ind_row.size, _pi(ind_chr), ind_chr.size, _pd(_f64(pos_chr)),
                                          _pd(_f64(st["sumX"])), _pd(_f64(st["denoX"])), len(sub_cols), _pi(lens),
                                          _pi(cat(sub_cols)), _pi(cat(sub_ords)), npt, _pd(_f64(p_thr)), _pd(_f64(p_size)),
                                          _pi(keep)))
        res, o = [], 0
        for sub in sub_cols:
            for _ in range(npt):
                k = keep[o:o + sub.size]
                res.append(ind_chr[sub[k == 1]])
                o += sub.size
        out.append(res)
    out.grid = grid
    return out


def prod_and_rowSumsSq(obj_bed, ind_row, ind_col, center, scale, V):
    """src/bed-fun.cpp:103-133 -> (XV (nr, K), rowSumsSq (nr)); V has one row per selected column (:116)."""
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    center, scale = _f64(center), _f64(scale)
    V = np.asarray(V, dtype=np.float64)
    V = np.asfortranarray(V.reshape(V.shape[0], -1))
    if center.size != ind_col.size or scale.size != ind_col.size or V.shape[0] != ind_col.size:
        raise ValueError(ERROR_DIM)
    K = V.shape[1]
    XV = np.empty((ind_row.size, K), dtype=np.float64, order="F")
    rss = np.empty(ind_row.size, dtype=np.float64)
    check(lib().bsg_prod_and_rowsumssq(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                                       _pd(scale), V.ctypes.data_as(_lib.c_dbl_p), K,
                                       XV.ctypes.data_as(_lib.c_dbl_p), _pd(rss)))
    return XV, rss


def prod_and_rowSumsSq2(G, ind_row, ind_col, center, scale, V):
    """src/project-utils.cpp:11-43 on an FBM.code256 handle -> (XV (nr, K), rowSumsSq (nr)); an NA code is NA_real, so a
    row holding one in a selected column is NaN in both outputs."""
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    center, scale = _f64(center), _f64(scale)
    V = np.asarray(V, dtype=np.float64)
    V = np.asfortranarray(V.reshape(V.shape[0], -1))
    if center.size != ind_col.size or scale.size != ind_col.size or V.shape[0] != ind_col.size:
        raise ValueError(ERROR_DIM)
    K = V.shape[1]
    XV = np.empty((ind_row.size, K), dtype=np.float64, order="F")
    rss = np.empty(ind_row.size, dtype=np.float64)
    check(lib().bsg_prod_and_rowsumssq2(G._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                                        _pd(scale), V.ctypes.data_as(_lib.c_dbl_p), K,
                                        XV.ctypes.data_as(_lib.c_dbl_p), _pd(rss)))
    return XV, rss


def snp_projectSelfPCA(obj_svd, G, ind_row, ind_col=None, ncores=1):
    """R/bed-projectPCA.R:252-281: project the samples `ind_row` of the FBM.code256 `G` on the PCs of `obj_svd` (dict with
    v, d, center, scale; `ind_col` defaults to its "subset").  Returns obj.svd.ref, simple_proj (= XV) and X_norm (row sums
    of squares); the OADP correction is bigutilsr::pca_OADP_proj2 on the host (un-vendored R code), as bed_projectSelfPCA."""
    v = np.asarray(obj_svd["v"], dtype=np.float64)
    if ind_col is None:
        ind_col = obj_svd.get("subset", None)
    if ind_col is None:
        raise ValueError("'ind.col' can't be `NULL`.")
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    _assert_lengths(np.arange(v.shape[0]), ind_col)
    XV, x_norm = prod_and_rowSumsSq2(G, ind_row, ind_col, obj_svd["center"], obj_svd["scale"], v)
    return {"obj.svd.ref": obj_svd, "simple_proj": XV, "X_norm": x_norm}


def bed_projectSelfPCA(obj_svd, obj_bed, ind_row, ind_col=None, ncores=1):
    """R/bed-projectPCA.R:196-227: project the samples `ind_row` of the same file on the PCs of `obj_svd`
    (dict with v, d, center, scale).  Returns obj.svd.ref, simple_proj (= XV) and X_norm (row sums of squares);
    the OADP correction is bigutilsr::pca_OADP_proj2 applied to (XV, X_norm, d) on the host (un-vendored R code)."""
    _assert_bed(obj_bed)
    v = np.asarray(obj_svd["v"], dtype=np.float64)
    if ind_col is None:
        ind_col = obj_svd.get("subset", None)
    if ind_col is None:
        raise ValueError("'ind.col' can't be `NULL`.")
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    _assert_lengths(np.arange(v.shape[0]), ind_col)
    XV, x_norm = prod_and_rowSumsSq(obj_bed, ind_row, ind_col, obj_svd["center"], obj_svd["scale"], v)
    return {"obj.svd.ref": obj_svd, "simple_proj": XV, "X_norm": x_norm}


def multLinReg(obj, ind_row, ind_col, U, ncores=1):
    """src/multLinReg.cpp:64-88 -> t-scores (nc, K), NaN where the reference gives NA."""
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    U = np.asarray(U, dtype=np.float64)
    U = np.asfortranarray(U.reshape(U.shape[0], -1))
    if U.shape[0] != ind_row.size:
        raise ValueError(ERROR_DIM)
    K = U.shape[1]
    out = np.empty((ind_col.size, K), dtype=np.float64, order="F")
    check(lib().bsg_multlinreg(obj._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size,
                               U.ctypes.data_as(_lib.c_dbl_p), K, out.ctypes.data_as(_lib.c_dbl_p)))
    return out


def bed_pcadapt(obj_bed, U_row, ind_row=..., ind_col=..., ncores=1):
    """R/pcadapt.R:3-27,73-81 up to the t-scores: the Mahalanobis distance (bigutilsr::dist_ogk) and the genomic
    control that follow are host-side R code on the (nc x K) matrix returned here.  K == 1 returns the reference's
    score (t - median(t))^2 directly."""
    _assert_bed(obj_bed)
    ind_row, ind_col = _ind(obj_bed, *_dflt(obj_bed, ind_row, ind_col))
    U = np.asarray(U_row, dtype=np.float64)
    U = U.reshape(U.shape[0], -1)
    _assert_lengths(np.arange(U.shape[0]), ind_row)
    t = multLinReg(obj_bed, ind_row, ind_col, U, ncores)
    if U.shape[1] == 1:
        return {"tscores": t, "score": (t[:, 0] - np.median(t[:, 0])) ** 2}
    return {"tscores": t}


snp_pcadapt = bed_pcadapt  # R/pcadapt.R:61-68 (FBM.code256 handles share the packed kernels)


def readbina2(obj_bed, ind_row, ind_col, ncores=1):
    """src/read-plink.cpp:61-80 -> the FBM.code256 bytes (nr, nc) uint8 with codes 0 / 1 / 2 / 3 (NA)."""
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    out = np.empty((ind_row.size, ind_col.size), dtype=np.uint8, order="F")
    check(lib().bsg_readbina2(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size,
                              out.ctypes.data_as(C.POINTER(C.c_uint8))))
    return out


def snp_readBed2(bedfile, backingfile=None, ind_row=..., ind_col=..., ncores=1):
    """R/read-plink.R:72-111: fill an FBM.code256 (code CODE_012) from a .bed.  Returns dict(genotypes = (nr, nc) uint8
    codes, map = the selected .bim rows, backingfile); with `backingfile` the bytes are also written to
    `<backingfile>.bk` (column-major, the FBM layout), refusing to overwrite like assert_noexist."""
    obj = bed(bedfile)
    try:
        ind_row, ind_col = _ind(obj, *_dflt(obj, ind_row, ind_col))
        G = readbina2(obj, ind_row, ind_col, ncores)
        bim = {k: np.asarray(v)[ind_col - 1] for k, v in obj.map.items()}
    finally:
        obj.close()
    bk = None
    if backingfile is not None:
        bk = os.path.expanduser(backingfile) + ".bk"
        if os.path.exists(bk):
            raise FileExistsError("File '%s' already exists." % bk)
        G.T.tofile(bk)  # column-major on disk
    return {"genotypes": G, "map": bim, "backingfile": bk}


def writebina(filename, obj, ind_row, ind_col):
    """src/write-plink.cpp:13-52: X[ind_row, ind_col] of a staged handle as a .bed file (the reference's bytes)."""
    ind_row, ind_col = _i32(ind_row), _i32(ind_col)
    check(lib().bsg_writebina(obj._h, os.fsencode(filename), _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size))


def snp_writeBed(G, bedfile, ind_row=..., ind_col=...):
    """R/write-plink.R:15-45 for the genotype part: write `bedfile` from a handle (bed- or FBM.code256-staged).
    The .bim / .fam tables are plain-text host data of the caller's bigSNP and are not produced here."""
    if os.path.exists(bedfile):
        raise FileExistsError("File '%s' already exists." % bedfile)
    os.makedirs(os.path.dirname(os.path.abspath(bedfile)), exist_ok=True)
    ind_row, ind_col = _ind(G, *_dflt(G, ind_row, ind_col))
    writebina(os.path.expanduser(bedfile), G, ind_row, ind_col)
    return bedfile


def bed_clumping_chr(obj_bed, ind_row, ind_col, center, scale, ordInd, rankInd, pos, size, thr, ncores=1):
    """src/clumping-bed.cpp:11-91 -> keep (int32 0/1 per column of ind_col).  rankInd is implied by ordInd."""
    ind_row, ind_col, ordInd = _i32(ind_row), _i32(ind_col), _i32(ordInd)
    center, scale, pos = _f64(center), _f64(scale), _f64(pos)
    for v in (center, scale, pos, ordInd):
        if v.size != ind_col.size:
            raise ValueError(ERROR_DIM)
    keep = np.full(ind_col.size, -1, dtype=np.int32)
    check(lib().bsg_clumping_chr(obj_bed._h, _pi(ind_row), ind_row.size, _pi(ind_col), ind_col.size, _pd(center),
                                 _pd(scale), _pi(ordInd), _pd(pos), float(size), float(thr), _pi(keep)))
    return keep


def bed_clumping(obj_bed, ind_row=..., S=None, thr_r2=0.2, size=None, exclude=None, ncores=1, infos_chr=None,
                 infos_pos=None):
    """LD clumping on a bed object (R/bed-clumping.R:7-74): sorted 1-based indices of the variants kept."""
    _assert_bed(obj_bed)
    if ind_row is None:
        raise ValueError("'ind.row' can't be `NULL`.")
    ind_row = obj_bed.rows_along() if ind_row is ... else _i32(ind_row)
    if size is None:
        size = 100 / thr_r2
    if infos_chr is None:
        infos_chr = obj_bed.map["chromosome"]
    if infos_pos is None:
        infos_pos = obj_bed.map["physical.pos"]
    infos_chr, infos_pos = np.asarray(infos_chr), _f64(infos_pos)
    m = obj_bed.ncol
    if S is not None:
        _assert_lengths(infos_chr, S)
    noexcl = np.setdiff1d(np.arange(1, m + 1), np.asarray([] if exclude is None else exclude, dtype=np.int64))
    kept = []
    for chrom in sorted(set(infos_chr[noexcl - 1].tolist())):
        ind_chr = noexcl[infos_chr[noexcl - 1] == chrom].astype(np.int32)
        st = bed_colstats(obj_bed, ind_row, ind_chr, ncores)
        with np.errstate(all="ignore"):
            center = st["sumX"] / st["nb_nona_col"]
            scale = np.sqrt(st["denoX"])
        S_chr = np.minimum(st["sumX"], 2 * st["nb_nona_col"] - st["sumX"]) if S is None else np.asarray(S)[ind_chr - 1]
        ordv = (np.argsort(-np.asarray(S_chr, dtype=np.float64), kind="stable") + 1).astype(np.int32)
        pos_chr = infos_pos[ind_chr - 1]
        if np.any(np.diff(pos_chr) < 0):
            raise ValueError("'pos.chr' is not sorted.")
        keep = bed_clumping_chr(obj_bed, ind_row, ind_chr, center, scale, ordv, None, pos_chr, size * 1000.0, thr_r2, ncores)
        if not np.all((keep == 0) | (keep == 1)):
            raise RuntimeError("clumping left undecided variants")
        kept.append(ind_chr[keep == 1])
    return np.sort(np.concatenate(kept)) if kept else np.zeros(0, dtype=np.int32)


# ---- sparse LD matrix (bigsparser's SFBM) and lassosum2 -------------------------------------------------------------------

def _full_columns(n, p, i, x, upper):
    """CSC (p, i, x) of an n x n matrix -> the full symmetric CSC (rows ascending per column), stored entries kept as they
    are (explicit zeros included).  upper: (p, i, x) holds the upper triangle with the diagonal, mirrored here."""
    import scipy.sparse as sp

    # canonical order: rows ascending within each column, repeated (row, column) entries summed
    a = sp.csc_matrix((np.array(x, dtype=np.float64), np.array(i, dtype=np.int64), np.array(p, dtype=np.int64)),
                      shape=(n, n))  # copies: the caller's arrays stay as they are
    a.sum_duplicates()
    p, i, x = a.indptr.astype(np.int64), a.indices.astype(np.int64), a.data
    if not upper:
        return p, i, x
    cnt = np.diff(p)
    col = np.repeat(np.arange(n, dtype=np.int64), cnt)
    if np.any(i > col):
        raise ValueError("'corr' is flagged upper-triangular but stores entries below the diagonal.")
    # the transpose holds, per column j, the rows >= j in ascending order: its diagonal entry (if any) comes first
    lt = sp.csc_matrix((x, i, p), shape=(n, n)).T.tocsc()
    lt.has_sorted_indices = False
    lt.sort_indices()
    lp, li, lx = lt.indptr.astype(np.int64), lt.indices.astype(np.int64), lt.data
    has_diag = np.zeros(n, dtype=bool)
    nz = cnt > 0
    has_diag[nz] = i[p[1:][nz] - 1] == np.arange(n)[nz]
    cnt_l = np.diff(lp) - has_diag
    fp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(cnt + cnt_l, out=fp[1:])
    fi, fx = np.empty(fp[-1], dtype=np.int64), np.empty(fp[-1])
    dest = fp[col] + (np.arange(p[-1], dtype=np.int64) - p[col])  # the upper part (with the diagonal) first
    fi[dest], fx[dest] = i, x
    lcol = np.repeat(np.arange(n, dtype=np.int64), np.diff(lp))
    k = np.arange(lp[-1], dtype=np.int64) - lp[lcol]
    strict = li > lcol
    dest = fp[lcol] + cnt[lcol] + k - has_diag[lcol]  # then the rows below the diagonal
    fi[dest[strict]], fx[dest[strict]] = li[strict], lx[strict]
    return fp, fi, fx


def sfbm_storage(corr, compact=False, upper=None):
    """bigsparser's storage of as_SFBM(corr, compact) as bigsnpr reads it (src/ld-scores-sfbm.cpp:14-66), built on the
    host: (n, p, data, first_i) with p the ncol + 1 offsets as doubles; non-compact data interleaves (row, value) doubles
    and first_i is None; compact data holds values only, column j running from its smallest stored row first_i[j] to its
    largest with zeros filled in (an empty column: first_i 0, no value).

    corr: the (p, i, x) tuple of bed_cor / snp_cor (the upper triangle with the diagonal, expanded to full columns), or a
    square scipy.sparse matrix, symmetric as stored unless `upper=True` flags an upper-triangular one."""
    if isinstance(corr, tuple):
        p, i, x = corr
        n = len(p) - 1
        upper = True if upper is None else upper
    else:
        import scipy.sparse as sp

        if not sp.issparse(corr):
            raise TypeError("'corr' must be the (p, i, x) tuple of bed_cor or a scipy.sparse matrix.")
        if corr.shape[0] != corr.shape[1]:
            raise ValueError(ERROR_DIM)
        a = sp.csc_matrix(corr, dtype=np.float64, copy=True)
        a.sum_duplicates()
        n, p, i, x = a.shape[0], a.indptr, a.indices, a.data
        upper = bool(upper)
    p, i, x = _full_columns(n, p, i, x, upper)
    if not compact:
        data = np.empty(2 * x.size)
        data[0::2], data[1::2] = i, x
        return n, p.astype(np.float64), data, None
    cnt = np.diff(p)
    nz = cnt > 0
    first_i = np.zeros(n, dtype=np.int32)
    lens = np.zeros(n, dtype=np.int64)
    first_i[nz] = i[p[:-1][nz]]
    lens[nz] = i[p[1:][nz] - 1] - first_i[nz] + 1
    cp = np.zeros(n + 1, dtype=np.int64)
    np.cumsum(lens, out=cp[1:])
    data = np.zeros(cp[-1])
    col = np.repeat(np.arange(n, dtype=np.int64), cnt)
    data[cp[col] + (i - first_i[col])] = x
    return n, cp.astype(np.float64), data, first_i


class SFBM:
    """as_SFBM(corr, compact) on the device (bsg_sfbm_open): the sparse LD matrix snp_lassosum2 and ld_scores_sfbm read.
    Keeps the host storage arrays `p`, `data` and `first_i` (None when not compact), as the R object exposes them."""

    def __init__(self, nrow, ncol, p, data, first_i=None, device=0):
        self.p, self.data = _f64(p), _f64(data)
        self.first_i = None if first_i is None else _i32(first_i)
        self.compact = first_i is not None
        h = _lib.vp()
        check(lib().bsg_sfbm_open(int(nrow), int(ncol), _pd(self.p), _pd(self.data), _pi(self.first_i), int(device),
                                  C.byref(h)))
        self._h = h

    @property
    def nrow(self):
        return lib().bsg_sfbm_nrow(self._h)

    @property
    def ncol(self):
        return lib().bsg_sfbm_ncol(self._h)

    @property
    def shape(self):
        return (self.nrow, self.ncol)

    def cols_along(self):
        return np.arange(1, self.ncol + 1, dtype=np.int32)

    def close(self):
        if getattr(self, "_h", None):
            lib().bsg_sfbm_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown
            pass


def as_SFBM(corr, compact=False, upper=None, device=0):
    """bigsparser::as_SFBM: the sparse LD matrix resident on the device.  corr: the (p, i, x) tuple of bed_cor / snp_cor, or
    a scipy.sparse matrix (symmetric, or upper-triangular flagged with upper=True).  See sfbm_storage."""
    n, p, data, first_i = sfbm_storage(corr, compact, upper)
    return SFBM(n, n, p, data, first_i, device)


def ld_scores_sfbm(corr, ind_corr=None, ncores=1):
    """src/ld-scores-sfbm.cpp:9-69: per column ind_corr[j] (1-based like the rest of this module; default all), the sum of
    the squared stored values whose row is in ind_corr.  The .Call target receives ind_corr - 1, as here."""
    ind_sub = np.arange(corr.ncol, dtype=np.int32) if ind_corr is None else _i32(np.asarray(ind_corr) - 1)
    out = np.empty(ind_sub.size)
    check(lib().bsg_sfbm_ld_scores(corr._h, _pi(ind_sub), ind_sub.size, _pd(out)))
    return out


def seq_log(from_, to, length_out):
    """R/SCT.R:167-171: exp(seq(log(from), log(to), length.out)), with seq's rule for the points (both ends exact, the
    inner ones from + i * by) and the C library's exp."""
    import math

    n = int(length_out)
    a, b = math.log(from_), math.log(to)
    if n <= 2:
        s = np.array([a, b][:n])
    elif a == b:
        s = np.full(n, a)
    else:
        s = np.concatenate([[a], a + np.arange(1, n - 1) * ((b - a) / (n - 1)), [b]])
    return np.array([math.exp(v) for v in s])


class Lassosum2Grid(np.ndarray):
    """snp_lassosum2's result: the m x ngrid matrix of effects with the `grid_param` attribute (dict of columns lambda,
    delta, num_iter, time, sparsity, one row per column of the matrix)."""

    grid_param = None


def _df_column(df, name, what="df_beta"):
    try:
        if name in df:
            return _f64(df[name])
    except TypeError:
        pass
    raise ValueError("'%s' should have element '%s'." % (what, name))


def _lassosum2_grid(beta, beta_se, n_eff, delta, nlambda, lambda_min_ratio):
    """R/lassosum2.R:40-51 and the arguments of every lassosum2 call (:58-67): (beta_hat, scale, lambda and delta of each
    grid point in expand.grid order, lambda fastest, then the m x ngrid lambda and delta_plus_one matrices)."""
    N = n_eff
    scale = np.sqrt(N * beta_se ** 2 + beta ** 2)
    beta_hat = beta / scale
    pf = np.sqrt(np.max(N) / N)
    lambda0 = np.max(np.abs(beta_hat / pf))
    seq_lam = seq_log(lambda0, lambda_min_ratio * lambda0, nlambda + 1)[1:]
    g_lam, g_delta = np.tile(seq_lam, delta.size), np.repeat(delta, seq_lam.size)
    lam = np.asfortranarray(pf[:, None] * g_lam[None, :])
    dp1 = np.asfortranarray(pf[:, None] * g_delta[None, :] + 1)
    return beta_hat, scale, g_lam, g_delta, lam, dp1


def snp_lassosum2(corr, df_beta, delta=(0.001, 0.01, 0.1, 1), nlambda=30, lambda_min_ratio=0.01, dfmax=200e3, maxiter=1000,
                  tol=1e-5, ind_corr=None, ncores=1):
    """R/lassosum2.R:25-81.  corr: an SFBM (as_SFBM); df_beta: a mapping (dict, data frame) with beta, beta_se and n_eff;
    ind_corr: 1-based columns of corr, one per row of df_beta.  The whole expand.grid(lambda, delta) grid (lambda fastest)
    runs in one bsg_lassosum2 call, one device CTA per point.  Returns the m x ngrid effects times `scale`, with
    `grid_param`."""
    if not hasattr(df_beta, "__getitem__") or not hasattr(df_beta, "__contains__"):
        raise TypeError("'df_beta' is not of class 'data.frame'.")
    beta, beta_se, n_eff = (_df_column(df_beta, k) for k in ("beta", "beta_se", "n_eff"))
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    ind_corr = corr.cols_along() if ind_corr is None else _i32(ind_corr)
    _assert_lengths(ind_corr, beta)
    if np.any((ind_corr < 1) | (ind_corr > corr.ncol)):
        raise ValueError("all(ind.corr %in% cols_along(corr)) is not TRUE")
    if not np.all(beta_se > 0):
        raise ValueError("'df_beta$beta_se' should have only positive values.")
    delta = _f64(np.asarray(delta, dtype=np.float64).reshape(-1))
    if not np.all(delta > 0):
        raise ValueError("'delta' should have only positive values.")
    beta_hat, scale, g_lam, g_delta, lam, dp1 = _lassosum2_grid(beta, beta_se, n_eff, delta, nlambda, lambda_min_ratio)
    m, ngrid = beta.size, g_lam.size
    beta_est = np.empty((m, ngrid), order="F")
    num_iter = np.empty(ngrid, dtype=np.int32)
    secs = np.empty(ngrid)
    ind_sub = _i32(ind_corr - 1)
    check(lib().bsg_lassosum2(corr._h, _pd(_f64(beta_hat)), m, _pi(ind_sub), ngrid, _pd(lam), _pd(dp1), float(dfmax),
                              int(maxiter), float(tol), _pd(beta_est), _pi(num_iter), _pd(secs)))
    sparsity = np.where(np.isnan(beta_est).any(axis=0), np.nan, (beta_est == 0).mean(axis=0))  # colMeans(beta == 0)
    with np.errstate(invalid="ignore"):  # a diverged point's NA column times scale
        out = np.asfortranarray(beta_est * scale[:, None]).view(Lassosum2Grid)
    out.grid_param = {"lambda": g_lam, "delta": g_delta, "num_iter": num_iter, "time": secs, "sparsity": sparsity}
    return out


# ---- LDpred2-inf (sp_solve_sym) and LD score regression --------------------------------------------------------------------

def _sp_solve(corr, b, add_to_diag, tol, maxiter):
    """bsg_sfbm_solve: (x, iters, error) of the conjugate-gradient solve of (corr + diag(add_to_diag)) x = b."""
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    b = _f64(np.asarray(b, dtype=np.float64).reshape(-1))
    d = _f64(np.asarray(add_to_diag, dtype=np.float64).reshape(-1))
    n = corr.ncol
    _assert_lengths(b, range(n))
    if d.size not in (1, n):
        raise ValueError(ERROR_DIM)
    maxiter = 10 * n if maxiter is None else int(maxiter)
    x = np.empty(n)
    it, err = C.c_int(), C.c_double()
    check(lib().bsg_sfbm_solve(corr._h, _pd(b), _pd(d), d.size, float(tol), maxiter, _pd(x), C.byref(it), C.byref(err)))
    return x, it.value, err.value


def sp_solve_sym(corr, b, add_to_diag=0, tol=1e-10, maxiter=None):
    """bigsparser::sp_solve_sym: x solving (corr + diag(add_to_diag)) x = b by the conjugate gradient on the device
    (bsg_sfbm_solve).  corr: an SFBM; add_to_diag: one value or one per column; maxiter None is 10 * ncol(corr).  A NaN
    error raises "Solver failed."; an error above tol warns "Estimated error: <error>."."""
    x, _, err = _sp_solve(corr, b, add_to_diag, tol, maxiter)
    if np.isnan(err):
        raise RuntimeError("Solver failed.")
    if err > tol:
        import warnings

        warnings.warn("Estimated error: %g." % err)
    return x


def snp_ldpred2_inf(corr, df_beta, h2):
    """R/LDpred2.R:27-42: effects under the infinitesimal model, x * scale with x solving
    (corr + diag(ncol / (h2 * N))) x = beta / scale, scale = sqrt(N * beta_se^2 + beta^2), N = n_eff."""
    if not hasattr(df_beta, "__getitem__") or not hasattr(df_beta, "__contains__"):
        raise TypeError("'df_beta' is not of class 'data.frame'.")
    beta, beta_se, n_eff = (_df_column(df_beta, k) for k in ("beta", "beta_se", "n_eff"))
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    _assert_lengths(range(corr.nrow), range(corr.ncol))
    _assert_lengths(range(corr.ncol), beta)
    if not np.all(beta_se > 0):
        raise ValueError("'df_beta$beta_se' should have only positive values.")
    h2 = np.asarray(h2, dtype=np.float64)
    if not np.all(h2 > 0):
        raise ValueError("'h2' should have only positive values.")
    N = n_eff
    scale = np.sqrt(N * beta_se ** 2 + beta ** 2)
    beta_hat = beta / scale
    beta_inf = sp_solve_sym(corr, beta_hat, add_to_diag=corr.ncol / (h2 * N))
    return beta_inf * scale


# ---- LDpred2-auto -------------------------------------------------------------------------------------------------------

_MRG_M1, _MRG_M2 = 4294967087, 4294944443


def _mrg_matpow(A, e, m):
    """A^e mod m for a 3 x 3 matrix of Python ints."""
    R = [[int(i == j) for j in range(3)] for i in range(3)]
    while e:
        if e & 1:
            R = [[sum(R[i][k] * A[k][j] for k in range(3)) % m for j in range(3)] for i in range(3)]
        A = [[sum(A[i][k] * A[k][j] for k in range(3)) % m for j in range(3)] for i in range(3)]
        e >>= 1
    return R


_MRG_A1 = [[0, 1, 0], [0, 0, 1], [_MRG_M1 - 810728, 1403580, 0]]
_MRG_A2 = [[0, 1, 0], [0, 0, 1], [_MRG_M2 - 1370589, 0, 527612]]
_MRG_J1, _MRG_J2 = _mrg_matpow(_MRG_A1, 2 ** 127, _MRG_M1), _mrg_matpow(_MRG_A2, 2 ** 127, _MRG_M2)


def mrg32k3a_next_stream(state):
    """The MRG32k3a state 2^127 draws further (parallel::nextRNGStream): the start of the next stream."""
    s = [int(v) for v in state]
    a = [sum(_MRG_J1[i][k] * s[k] for k in range(3)) % _MRG_M1 for i in range(3)]
    b = [sum(_MRG_J2[i][k] * s[3 + k] for k in range(3)) % _MRG_M2 for i in range(3)]
    return np.array(a + b, dtype=np.uint32)


def mrg32k3a_seed(seed):
    """The first MRG32k3a state of `seed` (an integer taken mod 2^32): x <- 69069 x + 1 (mod 2^32) applied 50 times, then
    once more for each of the six words, again while the word is not below m2."""
    x = int(seed) & 0xFFFFFFFF
    for _ in range(50):
        x = (69069 * x + 1) & 0xFFFFFFFF
    out = []
    for _ in range(6):
        x = (69069 * x + 1) & 0xFFFFFFFF
        while x >= _MRG_M2:
            x = (69069 * x + 1) & 0xFFFFFFFF
        out.append(x)
    return np.array(out, dtype=np.uint32)


def _ldpred2_auto_call(corr, beta_hat, n_vec, log_var, ind_sub, p_init, h2_init, burn_in, num_iter, report_step,
                       no_jump_sign, shrink_corr, use_mle, p_bounds, alpha_bounds, mean_ld, rng_state, sample=True,
                       rng_out=False):
    """bsg_ldpred2_auto_ex: a dict of the m x nchain estimates, the (burn_in + num_iter) x nchain paths, the dense
    m x n_reports x nchain sample_beta (None unless `sample`), each chain's device seconds and, with `rng_out`, the
    nchain x 6 MRG32k3a states the chains end in ("rng_out")."""
    m, nchain = int(np.size(beta_hat)), int(np.size(p_init))
    T, nrep = int(burn_in) + int(num_iter), int(num_iter) // max(int(report_step), 1)
    rng = np.ascontiguousarray(np.asarray(rng_state, dtype=np.uint32).reshape(nchain * 6))
    est = [np.empty((m, nchain), order="F") for _ in range(3)]
    paths = [np.empty((T, nchain), order="F") for _ in range(3)]
    smp = np.empty((m, nrep, nchain), order="F") if sample else None
    secs = np.empty(nchain)
    rout = np.empty((nchain, 6), dtype=np.uint32) if rng_out else None
    check(lib().bsg_ldpred2_auto_ex(
        corr._h, _pd(_f64(beta_hat)), _pd(_f64(n_vec)), _pd(_f64(log_var)), m, _pi(_i32(ind_sub)), nchain,
        _pd(_f64(p_init)), float(h2_init), int(burn_in), int(num_iter), int(report_step), int(bool(no_jump_sign)),
        float(shrink_corr), int(bool(use_mle)), _pd(_f64(p_bounds)), _pd(_f64(alpha_bounds)), float(mean_ld),
        rng.ctypes.data_as(C.POINTER(C.c_uint)), *(_pd(a) for a in est), *(_pd(a) for a in paths),
        None if smp is None else _pd(smp), _pd(secs), None if rout is None else rout.ctypes.data_as(C.POINTER(C.c_uint))))
    out = dict(zip(("beta_est", "postp_est", "corr_est"), est))
    out.update(zip(("path_p_est", "path_h2_est", "path_alpha_est"), paths))
    out["sample_beta"], out["time"] = smp, secs
    if rng_out:
        out["rng_out"] = rout
    return out


def _mrg_streams(seed, n):
    """n MRG32k3a states: mrg32k3a_seed(seed), then each the previous jumped 2^127 draws (%dorng%'s streams)."""
    st, out = mrg32k3a_seed(seed), []
    for _ in range(n):
        out.append(st)
        st = mrg32k3a_next_stream(st)
    return np.array(out, dtype=np.uint32).reshape(n, 6)


def snp_ldpred2_auto(corr, df_beta, h2_init, vec_p_init=0.1, burn_in=500, num_iter=200, sparse=False, verbose=False,
                     report_step=None, allow_jump_sign=True, shrink_corr=1, use_MLE=True, p_bounds=(1e-5, 1),
                     alpha_bounds=(-1.5, 0.5), ind_corr=None, ncores=1, seed=None):
    """R/LDpred2.R:203-286: LDpred2-auto, every chain (one per vec_p_init) in one bsg_ldpred2_auto launch.

    corr: an SFBM; df_beta: a mapping with beta, beta_se and n_eff; ind_corr: 1-based columns of corr, one per row of
    df_beta (default all); report_step None is num_iter + 1.  Returns a list over vec_p_init (in its order) of dicts with
    beta_est (allele scale), postp_est, corr_est, sample_beta (scipy.sparse.csc_matrix, one row per row of df_beta as in
    the reference, num_iter // report_step columns, not on the allele scale), path_p_est, path_h2_est, path_alpha_est, h2_est, p_est, alpha_est,
    h2_init, p_init.

    The chains run in R's order(-vec_p_init) (large p first, ties in input order); the i-th of that order draws from the
    MRG32k3a stream mrg32k3a_seed(seed) jumped i x 2^127 draws (parallel::nextRNGStream's jump).  seed None takes one from
    NumPy's global generator.  The draws follow R's sampler but are not R's stream: see DESIGN.md §4.15.  The MLE step
    returns the minimiser of the reference's objective over its box, where R returns the point L-BFGS-B stops at.
    sparse=True is not served here: snp_ldpred2_grid runs the same sparse sampler (ldpred2_gibbs_one) with a chain's
    p_est and h2_est, on a stream of its own, and the C ABI's bsg_ldpred2_auto_ex / bsg_ldpred2_grid continue a chain's
    own stream as R/LDpred2.R:266-279 does (DESIGN.md §4.15)."""
    if sparse:
        raise NotImplementedError("sparse = TRUE is not served by snp_ldpred2_auto; run snp_ldpred2_grid with the chains' "
                                  "p_est and h2_est and sparse = TRUE.")
    if not hasattr(df_beta, "__getitem__") or not hasattr(df_beta, "__contains__"):
        raise TypeError("'df_beta' is not of class 'data.frame'.")
    beta, beta_se, n_eff = (_df_column(df_beta, k) for k in ("beta", "beta_se", "n_eff"))
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    ind_corr = corr.cols_along() if ind_corr is None else _i32(ind_corr)
    _assert_lengths(ind_corr, beta)
    if np.any((ind_corr < 1) | (ind_corr > corr.ncol)):
        raise ValueError("all(ind.corr %in% cols_along(corr)) is not TRUE")
    if not np.all(beta_se > 0):
        raise ValueError("'df_beta$beta_se' should have only positive values.")
    h2_init = float(h2_init)
    if not h2_init > 0:
        raise ValueError("'h2_init' should have only positive values.")
    num_iter, burn_in = int(num_iter), int(burn_in)
    report_step = num_iter + 1 if report_step is None else int(report_step)
    vec_p_init = _f64(np.asarray(vec_p_init, dtype=np.float64).reshape(-1))
    N = n_eff
    sd = 1 / np.sqrt(N * beta_se ** 2 + beta ** 2)
    beta_hat = beta * sd
    ind_sub = _i32(ind_corr - 1)
    mean_ld = float(np.mean(ld_scores_sfbm(corr, ind_corr)))
    ord_ = np.argsort(-vec_p_init, kind="stable")
    if seed is None:
        seed = int(np.random.randint(0, 2 ** 31 - 1))
    r = _ldpred2_auto_call(corr, beta_hat, N, 2 * np.log(sd), ind_sub, vec_p_init[ord_], h2_init, burn_in, num_iter,
                           report_step, not allow_jump_sign, shrink_corr, use_MLE, np.asarray(p_bounds, dtype=np.float64),
                           np.asarray(alpha_bounds, dtype=np.float64) + 1, mean_ld, _mrg_streams(seed, ord_.size),
                           sample=True)
    import scipy.sparse as sp

    res = [None] * ord_.size
    for i, c in enumerate(ord_):
        out = {"beta_est": r["beta_est"][:, i] / sd, "postp_est": r["postp_est"][:, i].copy(),
               "corr_est": r["corr_est"][:, i].copy()}
        out["sample_beta"] = sp.csc_matrix(r["sample_beta"][:, :, i])
        for k in ("path_p_est", "path_h2_est", "path_alpha_est"):
            out[k] = r[k][:, i].copy()
        tail = slice(out["path_h2_est"].size - num_iter, None)
        out["h2_est"] = float(np.mean(out["path_h2_est"][tail]))
        out["p_est"] = float(np.mean(out["path_p_est"][tail]))
        out["alpha_est"] = float(np.mean(out["path_alpha_est"][tail]))
        out["h2_init"], out["p_init"] = h2_init, float(vec_p_init[c])
        out["time"] = float(r["time"][i])
        res[c] = out
    return res


def _ldpred2_grid_call(corr, beta_hat, n_vec, ind_sub, p, h2, sparse, burn_in, num_iter, rng_state, sampling=False):
    """bsg_ldpred2_grid: a dict of the m x npoint beta_est (or, with `sampling`, the m x num_iter sample_beta of the one
    point) and each point's device seconds ("time"); point g runs with p[g], h2[g], sparse[g] on the MRG32k3a state
    rng_state[g]."""
    p, h2 = _f64(np.asarray(p, dtype=np.float64).reshape(-1)), _f64(np.asarray(h2, dtype=np.float64).reshape(-1))
    sparse = _i32(np.asarray(sparse).reshape(-1).astype(bool))
    m, npoint = int(np.size(beta_hat)), p.size
    rng = np.ascontiguousarray(np.asarray(rng_state, dtype=np.uint32).reshape(npoint * 6))
    est = None if sampling else np.empty((m, npoint), order="F")
    smp = np.empty((m, int(num_iter)), order="F") if sampling else None
    secs = np.empty(npoint)
    check(lib().bsg_ldpred2_grid(corr._h, _pd(_f64(beta_hat)), _pd(_f64(n_vec)), m, _pi(_i32(ind_sub)), npoint, _pd(p),
                                 _pd(h2), _pi(sparse), int(burn_in), int(num_iter), int(bool(sampling)),
                                 rng.ctypes.data_as(C.POINTER(C.c_uint)), None if est is None else _pd(est),
                                 None if smp is None else _pd(smp), _pd(secs)))
    return {"beta_est": est, "sample_beta": smp, "time": secs}


def _ldpred2_grid_order(p, h2, sparse):
    """R's order(-p, sparse, -h2): stable, large p first, then non-sparse first, then large h2 first."""
    return np.lexsort((-np.asarray(h2, dtype=np.float64), np.asarray(sparse).astype(bool),
                       -np.asarray(p, dtype=np.float64)))


def snp_ldpred2_grid(corr, df_beta, grid_param, burn_in=50, num_iter=100, ncores=1, return_sampling_betas=False,
                     ind_corr=None, seed=None):
    """R/LDpred2.R:73-140: LDpred2-grid, every row of grid_param in one bsg_ldpred2_grid launch.

    corr: an SFBM; df_beta: a mapping with beta, beta_se and n_eff; grid_param: a mapping with p, h2 and sparse (one
    value per grid point); ind_corr: 1-based columns of corr, one per row of df_beta (default all).  Returns the m x
    ngrid effects (one column per row of grid_param, in its order) times scale = sqrt(n_eff beta_se^2 + beta^2), a column
    of NA where the point diverged; with return_sampling_betas (one row of grid_param only), the m x num_iter sampling
    betas times scale.

    The points run in R's order(-p, sparse, -h2) (stable); the i-th of that order draws from the MRG32k3a stream
    mrg32k3a_seed(seed) jumped i x 2^127 draws, as snp_ldpred2_auto's chains do, and the sampling run from the first
    stream.  seed None takes one from NumPy's global generator.  The draws follow R's sampler but are not R's stream: see
    DESIGN.md §4.18."""
    if not hasattr(df_beta, "__getitem__") or not hasattr(df_beta, "__contains__"):
        raise TypeError("'df_beta' is not of class 'data.frame'.")
    beta, beta_se, n_eff = (_df_column(df_beta, k) for k in ("beta", "beta_se", "n_eff"))
    if not hasattr(grid_param, "__getitem__") or not hasattr(grid_param, "__contains__"):
        raise TypeError("'grid_param' is not of class 'data.frame'.")
    g_p, g_h2, g_sparse = (_df_column(grid_param, k, "grid_param") for k in ("p", "h2", "sparse"))
    if not (g_p.size == g_h2.size == g_sparse.size):
        raise ValueError(ERROR_DIM)
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    ind_corr = corr.cols_along() if ind_corr is None else _i32(ind_corr)
    _assert_lengths(ind_corr, beta)
    if np.any((ind_corr < 1) | (ind_corr > corr.ncol)):
        raise ValueError("all(ind.corr %in% cols_along(corr)) is not TRUE")
    if not np.all(beta_se > 0):
        raise ValueError("'df_beta$beta_se' should have only positive values.")
    if not np.all(g_h2 > 0):
        raise ValueError("'grid_param$h2' should have only positive values.")
    N = n_eff
    scale = np.sqrt(N * beta_se ** 2 + beta ** 2)
    beta_hat = beta / scale
    ind_sub = _i32(ind_corr - 1)
    if seed is None:
        seed = int(np.random.randint(0, 2 ** 31 - 1))
    if return_sampling_betas:
        if g_p.size != 1:
            raise ValueError("Only one set of parameters is allowed when using 'return_sampling_betas'.")
        r = _ldpred2_grid_call(corr, beta_hat, N, ind_sub, g_p, g_h2, g_sparse != 0, burn_in, num_iter,
                               _mrg_streams(seed, 1), sampling=True)
        return np.asfortranarray(r["sample_beta"] * scale[:, None])
    ord_ = _ldpred2_grid_order(g_p, g_h2, g_sparse != 0)
    r = _ldpred2_grid_call(corr, beta_hat, N, ind_sub, g_p[ord_], g_h2[ord_], g_sparse[ord_] != 0, burn_in, num_iter,
                           _mrg_streams(seed, ord_.size))
    beta_gibbs = np.empty_like(r["beta_est"])
    beta_gibbs[:, ord_] = r["beta_est"]  # res_list[inv_ord]
    with np.errstate(invalid="ignore"):  # a diverged point's NA column times scale
        return np.asfortranarray(beta_gibbs * scale[:, None])


def _wlm(x, y, w):
    """R/ldsc.R:11-22 (stats::lm.wfit(cbind(1, x), y, w)), in its formula order."""
    wx = w * x
    W, WX = np.sum(w), np.sum(wx)
    WY, WXX, WXY = np.dot(w, y), np.dot(wx, x), np.dot(wx, y)
    alpha = (WXX * WY - WX * WXY) / (W * WXX - WX ** 2)
    beta = (WXY * W - WX * WY) / (W * WXX - WX ** 2)
    return alpha, beta, x * beta + alpha


def _wlm_no_int(x, y, w):
    """R/ldsc.R:25-31 (stats::lm.wfit(as.matrix(x), y, w))."""
    wx = w * x
    beta = np.dot(wx, y) / np.dot(wx, x)
    return beta, x * beta


def _weights(pred, w_ld):
    return 1 / (pred ** 2 * w_ld)


def snp_ldsc(ld_score, ld_size, chi2, sample_size, blocks=200, intercept=None, chi2_thr1=30, chi2_thr2=np.inf, ncores=1):
    """R/ldsc.R:70-170, on the host: LD score regression with the two-step estimator.  blocks None: (int, h2); else a number
    of blocks of consecutive variants or a block label per variant, and the delete-a-block jackknife gives
    (int, int_se, h2, h2_se).  intercept None estimates it (step 1, variants with chi2 < chi2_thr1)."""
    chi2 = _f64(chi2) + 1e-8
    if not np.all(chi2 > 0):
        raise ValueError("'chi2' should have only positive values.")
    ld_score = _f64(ld_score)
    _assert_lengths(chi2, ld_score)
    ld_size = np.asarray(ld_size)
    if ld_size.size != 1:
        raise ValueError("'ld_size' should be of length 1.")
    if ld_size != np.trunc(ld_size):
        raise ValueError("'ld_size' should contain only integers.")
    ld_size = float(ld_size)
    M = chi2.size
    sample_size = _f64(np.asarray(sample_size, dtype=np.float64).reshape(-1))
    if sample_size.size == 1:
        sample_size = np.repeat(sample_size, M)
    else:
        _assert_lengths(sample_size, chi2)

    if blocks is None:
        if intercept is None:  # step 1
            ind_sub1 = chi2 < chi2_thr1
            w_ld = np.maximum(ld_score[ind_sub1], 1)
            x1 = (ld_score / ld_size * sample_size)[ind_sub1]
            y1 = chi2[ind_sub1]
            pred0 = y1
            for _ in range(100):
                pred = _wlm(x1, y1, _weights(pred0, w_ld))[2]
                if np.max(np.abs(pred - pred0)) < 1e-6:
                    break
                pred0 = pred
            step1_int = _wlm(x1, y1, _weights(pred0, w_ld))[0]
        else:
            step1_int = float(intercept)
        # step 2
        ind_sub2 = chi2 < chi2_thr2
        w_ld = np.maximum(ld_score[ind_sub2], 1)
        x = (ld_score / ld_size * sample_size)[ind_sub2]
        y = chi2[ind_sub2]
        yp = y - step1_int
        pred0 = y
        for _ in range(100):
            pred = step1_int + _wlm_no_int(x, yp, _weights(pred0, w_ld))[1]
            if np.max(np.abs(pred - pred0)) < 1e-6:
                break
            pred0 = pred
        step2_h2 = _wlm_no_int(x, yp, _weights(pred0, w_ld))[0]
        return np.array([step1_int, step2_h2])

    # delete-a-group jackknife (the fits receive chi2 + 1e-8, to which they add 1e-8 again, as the reference's do)
    blocks = np.asarray(blocks).reshape(-1)
    if blocks.size == 1:
        blocks = np.sort(np.resize(np.arange(1, int(blocks[0]) + 1), M))  # sort(rep_len(seq_len(blocks), M))
    else:
        _assert_lengths(blocks, chi2)
    labels = np.unique(blocks)
    ind_blocks = [np.flatnonzero(blocks == lab) for lab in labels]  # split(seq_along(blocks), blocks)
    h_blocks = M / np.array([ib.size for ib in ind_blocks], dtype=np.float64)
    fits = []
    for ind_rm in [None] + ind_blocks:
        keep = np.ones(M, dtype=bool)
        if ind_rm is not None:
            keep[ind_rm] = False
        fits.append(snp_ldsc(ld_score[keep], ld_size, chi2[keep], sample_size[keep], None, intercept, chi2_thr1,
                             chi2_thr2))
    delete_values = np.array(fits).T
    estim = delete_values[:, 0]
    int_pseudo = h_blocks * estim[0] - (h_blocks - 1) * delete_values[0, 1:]
    h2_pseudo = h_blocks * estim[1] - (h_blocks - 1) * delete_values[1, 1:]
    int_J = np.sum(int_pseudo / h_blocks)
    h2_J = np.sum(h2_pseudo / h_blocks)
    return np.array([int_J, np.sqrt(np.mean((int_pseudo - int_J) ** 2 / (h_blocks - 1))),
                     h2_J, np.sqrt(np.mean((h2_pseudo - h2_J) ** 2 / (h_blocks - 1)))])


def snp_ldsc2(corr, df_beta, blocks=None, intercept=1, ncores=1, ind_beta=None, chi2_thr1=30, chi2_thr2=np.inf):
    """R/ldsc.R:202-224 on an SFBM: snp_ldsc with the LD scores of ld_scores_sfbm over all columns, ld_size = ncol(corr),
    chi2 = (beta / beta_se)^2 and sample_size = n_eff.  ind_beta: 1-based columns of corr, one per row of df_beta."""
    if not hasattr(df_beta, "__getitem__") or not hasattr(df_beta, "__contains__"):
        raise TypeError("'df_beta' is not of class 'data.frame'.")
    beta, beta_se, n_eff = (_df_column(df_beta, k) for k in ("beta", "beta_se", "n_eff"))
    if not isinstance(corr, SFBM):
        raise TypeError("'corr' is not of class 'SFBM'.")
    ind_beta = corr.cols_along() if ind_beta is None else _i32(ind_beta)
    _assert_lengths(ind_beta, beta)
    if np.any((ind_beta < 1) | (ind_beta > corr.ncol)):
        raise ValueError("all(ind.beta %in% cols_along(corr)) is not TRUE")
    if not np.all(beta_se > 0):
        raise ValueError("'df_beta$beta_se' should have only positive values.")
    full_ld = ld_scores_sfbm(corr)
    return snp_ldsc(full_ld[ind_beta - 1], corr.ncol, (beta / beta_se) ** 2, n_eff, blocks=blocks, intercept=intercept,
                    chi2_thr1=chi2_thr1, chi2_thr2=chi2_thr2)


# ---- near-independent LD blocks (snp_ldsplit) ------------------------------------------------------------------------------

def ldsplit_lower(corr, upper=None):
    """Matrix::tril(corr) in CSC: (p int64, i int32, x float64), rows ascending within each column, repeated entries summed,
    explicit zeros kept.  corr: the (p, i, x) upper-triangle tuple of bed_cor / snp_cor (upper defaults to True), or a
    square scipy.sparse matrix, symmetric as stored unless `upper=True` flags an upper-triangular one (as in as_SFBM)."""
    import scipy.sparse as sp

    if isinstance(corr, tuple):
        p, i, x = corr
        n = len(p) - 1
        a = sp.csc_matrix((np.array(x, dtype=np.float64), np.array(i, dtype=np.int64), np.array(p, dtype=np.int64)),
                          shape=(n, n))
        upper = True if upper is None else upper
    else:
        if not sp.issparse(corr):
            raise TypeError("'corr' must be the (p, i, x) tuple of bed_cor or a scipy.sparse matrix.")
        if corr.shape[0] != corr.shape[1]:
            raise ValueError(ERROR_DIM)
        a = sp.csc_matrix(corr, dtype=np.float64, copy=True)
        upper = bool(upper)
    a.sum_duplicates()
    if upper:
        col = np.repeat(np.arange(a.shape[0]), np.diff(a.indptr))
        if np.any(a.indices > col):
            raise ValueError("'corr' is flagged upper-triangular but stores entries below the diagonal.")
        a = a.T.tocsc()
    else:
        a = sp.tril(a, format="csc")
    a.has_sorted_indices = False
    a.sort_indices()
    return a.indptr.astype(np.int64), a.indices.astype(np.int32), a.data.astype(np.float64)


def _ldsplit_args(m, min_size, max_size, max_K, max_cost, pos_scaled):
    """R/split-LD.R:105-106, plus max_size >= min_size and max_K >= 1: (max_size, pos_scaled, max_cost)."""
    max_size = np.atleast_1d(np.asarray(max_size))
    if max_size.size == 0 or not np.all(max_size == np.round(max_size)):
        raise ValueError("'max_size' must be whole numbers.")
    if not (min_size >= 1 and np.all(max_size <= m)):
        raise ValueError("min_size >= 1 && all(max_size <= m) is not TRUE")
    if np.any(max_size < min_size):
        raise ValueError("'max_size' must be at least 'min_size'.")
    if max_K < 1:
        raise ValueError("'max_K' must be at least 1.")
    pos = np.zeros(m) if pos_scaled is None else _f64(pos_scaled)
    _assert_lengths(pos, np.empty(m))
    return max_size, pos, (m / 200 if max_cost is None else float(max_cost))


def _check_diag(p, i, x):
    m = p.size - 1
    has = np.diff(p) > 0
    diag = np.zeros(m, dtype=bool)
    diag[has] = (i[p[:-1][has]] == np.arange(m)[has]) & (x[p[:-1][has]] != 0)
    if not np.all(diag):
        raise ValueError("all(Matrix::diag(corr) != 0) is not TRUE")


class LDCorr:
    """Matrix::tril(corr) resident on the device (bsg_ldcorr_open), the input of snp_ldsplit and get_L.  One handle
    serves any number of calls."""

    def __init__(self, corr, upper=None, device=0):
        self.p, self.i, self.x = ldsplit_lower(corr, upper) if not isinstance(corr, LDCorr) else (corr.p, corr.i, corr.x)
        self.m = self.p.size - 1
        if self.m < 1:
            raise ValueError("'corr' has no column.")
        _check_diag(self.p, self.i, self.x)
        h = _lib.vp()
        check(lib().bsg_ldcorr_open(self.m, self.p.ctypes.data_as(_lib.c_i64_p), _pi(self.i), _pd(self.x), int(device),
                                    C.byref(h)))
        self._h = h

    @property
    def sumsq2(self):
        return lib().bsg_ldcorr_sumsq2(self._h)

    def get_L(self, thr_r2, max_r2):
        """src/split-LD.cpp:15-61: dict of 0-based i (column of corr), j (row) and x, by column and row descending."""
        n = C.c_int64(0)
        check(lib().bsg_ldcorr_l_triplets(self._h, float(thr_r2), float(max_r2), C.byref(n), 0, None, None, None))
        li, lj, lx = np.empty(n.value, dtype=np.int32), np.empty(n.value, dtype=np.int32), np.empty(n.value)
        check(lib().bsg_ldcorr_l_triplets(self._h, float(thr_r2), float(max_r2), C.byref(n), n.value, _pi(li), _pi(lj), _pd(lx)))
        return {"i": li, "j": lj, "x": lx}

    def split(self, thr_r2, min_size, max_size, max_K=500, max_r2=0.3, max_cost=None, pos_scaled=None):
        """snp_ldsplit on this handle: (table or None, layers run per sorted max_size, device seconds of building E, of
        the layers and of the paths).  See snp_ldsplit."""
        m = self.m
        max_size, pos, max_cost = _ldsplit_args(m, min_size, max_size, max_K, max_cost, pos_scaled)
        S = _i32(max_size)
        ns, K = S.size, int(max_K)
        T = K * (K + 1) // 2
        kept = np.empty(ns * K, dtype=np.int32)
        cost, cost2, perc = np.empty(ns * K), np.empty(ns * K), np.empty(ns * K)
        path = np.empty(ns * T, dtype=np.int32)
        layers = np.empty(ns, dtype=np.int32)
        secs = np.empty(3)
        check(lib().bsg_ldsplit(self._h, float(thr_r2), int(min_size), _pi(S), ns, K, float(max_r2), max_cost, _pd(pos),
                                _pi(kept), _pd(cost), _pd(cost2), _pd(perc), _pi(path), _pi(layers), _pd(secs)))
        rows = np.flatnonzero(kept == 1)
        if rows.size == 0:
            return None, layers, secs
        t, nb = rows // K, rows % K + 1
        all_last = [path[tt * T + k * (k - 1) // 2: tt * T + k * (k + 1) // 2].copy() for tt, k in zip(t, nb)]
        table = {"max_size": np.sort(S)[t].astype(np.int32), "n_block": nb.astype(np.int32), "cost": cost[rows],
                 "cost2": cost2[rows], "perc_kept": perc[rows], "all_last": all_last,
                 "all_size": [np.diff(np.concatenate([[0], a])).astype(np.int32) for a in all_last]}
        return table, layers, secs

    def close(self):
        if getattr(self, "_h", None):
            lib().bsg_ldcorr_close(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:  # interpreter shutdown
            pass


def snp_ldsplit(corr, thr_r2, min_size, max_size, max_K=500, max_r2=0.3, max_cost=None, pos_scaled=None, upper=None):
    """R/split-LD.R:99-138: split a correlation matrix in near-independent blocks, for every max_size value (any order,
    run sorted).  corr: the (p, i, x) upper-triangle tuple of bed_cor, a scipy.sparse matrix (upper= as in as_SFBM), or
    an LDCorr handle.  max_cost defaults to m / 200 and is capped at 2 * sum(x^2) over the lower triangle (a sequential
    fold: R's BLAS crossprod can differ in the last bit).  The whole grid runs in one bsg_ldsplit call.  Returns None when
    no split is kept, else a dict of equal-length columns max_size, n_block, cost, cost2, perc_kept, all_last and
    all_size (the last two lists of int arrays, all_last 1-based)."""
    if not isinstance(corr, LDCorr):
        p, i, x = ldsplit_lower(corr, upper)
        _ldsplit_args(p.size - 1, min_size, max_size, max_K, max_cost, pos_scaled)
        _check_diag(p, i, x)
    h = corr if isinstance(corr, LDCorr) else LDCorr(corr, upper)
    try:
        return h.split(thr_r2, min_size, max_size, max_K, max_r2, max_cost, pos_scaled)[0]
    finally:
        if h is not corr:
            h.close()


def get_L(p, i, x, thr_r2, max_r2):
    """src/split-LD.cpp:15-61 on the lower triangle in CSC (p, i, x): dict of 0-based i, j and x triplets."""
    import scipy.sparse as sp

    n = len(p) - 1
    h = LDCorr(sp.csc_matrix((np.asarray(x, dtype=np.float64), np.asarray(i), np.asarray(p)), shape=(n, n)))
    try:
        return h.get_L(thr_r2, max_r2)
    finally:
        h.close()


def get_C(L, min_size, max_size, max_K, max_cost, pos_scaled, device=0):
    """src/split-LD.cpp:65-145: L is the m x (m + 1) scipy.sparse matrix built from get_L's triplets.  Returns a dict with
    C (m x max_K) and best_ind (1-based, NA_INTEGER where unset)."""
    import scipy.sparse as sp

    a = sp.csc_matrix(L, dtype=np.float64, copy=True)
    a.sum_duplicates()
    m = a.shape[0]
    if a.shape[1] != m + 1:
        raise ValueError(ERROR_DIM)
    pos = _f64(pos_scaled)
    _assert_lengths(pos, np.empty(m))
    K = int(max_K)
    Cm = np.empty((m, max(K, 0)), order="F")
    best = np.empty((m, max(K, 0)), dtype=np.int32, order="F")
    lp = a.indptr.astype(np.int64)
    check(lib().bsg_ldsplit_costs(m, lp.ctypes.data_as(_lib.c_i64_p), _pi(_i32(a.indices)), _pd(_f64(a.data)), int(min_size),
                                  int(max_size), K, float(max_cost), _pd(pos), int(device), _pd(Cm), _pi(best)))
    return {"C": Cm, "best_ind": best}


# ---- C+T scores (snp_PRS, snp_grid_PRS) -----------------------------------------------------------------------------------

class PRSScores(np.ndarray):
    """snp_PRS's result: the nr x nthr score matrix, with the thresholds as `thr_list` (R's column names)."""

    thr_list = None


class GridPRS(np.ndarray):
    """snp_grid_PRS's result: the nr x (keep sets x thresholds) score matrix (an np.memmap underneath when a backingfile
    was given), with the attributes lpS, grid_lpS_thr, betas and all_keep of R/SCT.R:239-245."""

    lpS = grid_lpS_thr = betas = all_keep = None


def _prs_call(G, ind_row, sets, beta_cat, same_cat, lpS_cat, thr, out):
    """One bsg_prs_grid call: keep sets `sets` (1-based column arrays) into the column-major block `out`."""
    lens = _i32([len(s) for s in sets])
    cols = _i32(np.concatenate([np.asarray(s).reshape(-1) for s in sets])) if sets else np.zeros(0, dtype=np.int32)
    same = None if same_cat is None else _i32(same_cat)
    lp = None if lpS_cat is None else _f64(lpS_cat)
    th = None if thr is None else _f64(thr)
    nthr = 1 if thr is None else th.size
    check(lib().bsg_prs_grid(G._h, _pi(ind_row), ind_row.size, len(sets), _pi(lens), _pi(cols), _pd(_f64(beta_cat)),
                             _pi(same), _pd(lp), nthr, _pd(th), int(out.dtype == np.float64),
                             C.c_void_p(out.ctypes.data) if out.size else None))


def _check_lpS(lpS, name):
    if np.any(np.isnan(lpS)):
        raise ValueError("%s must not have missing values." % name)
    if np.any(lpS < 0):
        raise ValueError("%s should have only non-negative values." % name)


def snp_PRS(G, betas_keep, ind_test=..., ind_keep=..., same_keep=None, lpS_keep=None, thr_list=0):
    """R/PRS.R:36-76 on a hard-call handle: the scores of ind_test for every threshold of thr_list (columns in the
    caller's order), one bsg_prs_grid call.  lpS_keep None or thr_list identical to 0: one column over every kept SNP."""
    import sys

    _assert_bed(G)
    ind_test = G.rows_along() if ind_test is ... else _i32(ind_test)
    ind_keep = G.cols_along() if ind_keep is ... else _i32(ind_keep)
    betas_keep = _f64(betas_keep)
    if same_keep is None:
        same_keep = np.ones(ind_keep.size, dtype=bool)
    else:
        same_keep = np.asarray(same_keep)
        if same_keep.dtype == object and any(s is None for s in same_keep.ravel()):
            raise ValueError("'same.keep' should have no missing value.")
        if same_keep.dtype != np.bool_:
            raise TypeError("'same.keep' should be of type 'logical'.")
    _assert_lengths(same_keep, ind_keep)
    _assert_lengths(betas_keep, ind_keep)
    thr = np.asarray(thr_list)
    disabled = lpS_keep is None or (thr.size == 1 and thr.dtype.kind in "if" and thr.item() == 0)
    if disabled:
        print("'lpS.keep' or 'thr.list' was not specified. Thresholding disabled.", file=sys.stderr)
        lp, th = None, None
    else:
        lp = _f64(lpS_keep)
        _assert_lengths(lp, ind_keep)
        _check_lpS(lp, "'lpS.keep'")
        th = _f64(thr.reshape(-1))
    out = np.empty((ind_test.size, 1 if th is None else th.size), order="F")
    _prs_call(G, ind_test, [ind_keep], betas_keep, same_keep.astype(np.int32), lp, th, out)
    out = out.view(PRSScores)
    out.thr_list = None if th is None else th
    return out


def snp_grid_PRS(G, all_keep, betas, lpS, n_thr_lpS=50, grid_lpS_thr=None, ind_row=..., backingfile=None, type="float",
                 ncores=1):
    """R/SCT.R:201-246: C+T scores of every keep set of snp_grid_clumping (a GridClumping, or a list per chromosome of
    1-based index arrays) at every threshold; column (ic - 1) n_thr + t is keep set ic (chromosome-major) at threshold t.
    One bsg_prs_grid call per chromosome.  backingfile: the matrix is an np.memmap of backingfile + '.bk' (R's FBM file)."""
    _assert_bed(G)
    betas, lpS = _f64(betas), _f64(lpS)
    _assert_lengths(G.cols_along(), betas)
    _assert_lengths(G.cols_along(), lpS)
    if type not in ("float", "double"):
        raise ValueError("'type' should be one of \"float\", \"double\".")
    if grid_lpS_thr is None:
        grid_lpS_thr = 0.9999 * seq_log(max(0.1, float(np.nanmin(lpS))), float(np.nanmax(lpS)), n_thr_lpS)
    thr = _f64(np.asarray(grid_lpS_thr, dtype=np.float64).reshape(-1))
    disabled = thr.size == 1 and thr[0] == 0  # snp_PRS's identical(thr.list, 0): one column over every kept SNP
    ind_row = G.rows_along() if ind_row is ... else _i32(ind_row)
    chroms = [[np.asarray(s, dtype=np.int64).reshape(-1) for s in chrom] for chrom in all_keep]
    cats = []
    for chrom in chroms:  # every chromosome is checked before the result file is created
        cat = np.concatenate(chrom) if chrom else np.zeros(0, dtype=np.int64)
        if np.any((cat < 1) | (cat > G.ncol)):
            raise IndexError("subscript out of bounds")
        if not disabled:
            _check_lpS(lpS[cat - 1], "'lpS.keep'")
        cats.append(cat)
    nsets = sum(len(c) for c in chroms)
    shape = (ind_row.size, nsets * thr.size)
    dtype = np.float32 if type == "float" else np.float64
    if backingfile is None:
        out = np.empty(shape, dtype=dtype, order="F")
    else:
        out = np.memmap(backingfile + ".bk", dtype=dtype, mode="w+", shape=shape, order="F")
    col = 0
    for chrom, cat in zip(chroms, cats):
        if not chrom:
            continue
        ncol = len(chrom) * thr.size
        _prs_call(G, ind_row, chrom, betas[cat - 1], None, None if disabled else lpS[cat - 1], None if disabled else thr,
                  out[:, col:col + ncol])
        col += ncol
    if backingfile is not None:
        out.flush()
    res = out.view(GridPRS)
    res.lpS, res.grid_lpS_thr, res.betas, res.all_keep = lpS, thr, betas, all_keep
    return res


class MHTest:
    """big_univLinReg's and big_univLogReg's result (bigstatsr's `mhtest` data frame): columns `estim`, `std_err`, `score`
    (in ind.col order), `transfo` = abs (what snp_clumping ranks on) and `predict`.  `df` is the t distribution's degrees
    of freedom; df = None means the normal distribution (big_univLogReg).  big_univLogReg also sets `niter` (IRLS steps,
    or glm.fit iterations for a refitted SNP) and `refitted` (the SNPs whose IRLS did not meet tol in maxiter steps)."""

    def __init__(self, estim, std_err, score, df, transfo=np.abs):
        self.estim, self.std_err, self.score, self.df, self.transfo = estim, std_err, score, df, transfo

    def __getitem__(self, name):
        return {"estim": self.estim, "std.err": self.std_err, "std_err": self.std_err, "score": self.score}[name]

    def __len__(self):
        return self.score.size

    def predict(self, log10=True):
        """log10 p-values of the two-sided test: (log 2 + log P(T > |score|)) / log 10 with T ~ t(df), or T ~ N(0, 1)
        when df is None; 10^that when log10 is False.  -predict() is snp_PRS's lpS."""
        from scipy import stats

        tail = stats.norm.logsf(np.abs(self.score)) if self.df is None else stats.t.logsf(np.abs(self.score), self.df)
        lp = (np.log(2) + tail) / np.log(10)
        return lp if log10 else 10 ** lp


def univlinreg_covar_basis(covar_train, n, thr_eigval=1e-4):
    """The R glue of big_univLinReg: U = the left singular vectors of cbind(1, covar.train) whose singular values, scaled
    by 1 / (sqrt(n) + sqrt(ncol) - 1), exceed thr_eigval (a duplicated column or a copy of the intercept drops out here)."""
    cols = [np.ones(n)]
    if covar_train is not None:
        cv = np.asarray(covar_train, dtype=np.float64)
        cols.append(cv.reshape(n, -1) if cv.ndim == 1 else cv)
    Cm = np.column_stack(cols)
    u, d, _ = np.linalg.svd(Cm, full_matrices=False)
    keep = d / (np.sqrt(n) + np.sqrt(Cm.shape[1]) - 1) > thr_eigval
    return np.asfortranarray(u[:, keep])


def big_univLinReg(X, y_train, ind_train=..., ind_col=..., covar_train=None, thr_eigval=1e-4, ncores=1):
    """bigstatsr's big_univLinReg on the device (bsg_univlinreg): the regression of y_train on [1, covar_train, X[, j]]
    for every column j of ind_col, in one pass over the matrix per 64 digit slices.  The SVD of the covariates, the choice
    of K and the degrees of freedom n - K - 1 run here in NumPy.  Returns an MHTest."""
    _assert_bed(X)
    ind_train = X.rows_along() if ind_train is ... else _i32(ind_train)
    ind_col = X.cols_along() if ind_col is ... else _i32(ind_col)
    y_train = _f64(y_train).reshape(-1)
    _assert_lengths(y_train, ind_train)
    n = ind_train.size
    if covar_train is not None:
        cv = np.asarray(covar_train, dtype=np.float64)
        if cv.shape[0] != n:
            raise ValueError(ERROR_DIM)
    U = univlinreg_covar_basis(covar_train, n, thr_eigval)
    K = U.shape[1]
    estim, std_err = np.empty(ind_col.size), np.empty(ind_col.size)
    check(lib().bsg_univlinreg(X._h, _pi(ind_train), n, _pi(ind_col), ind_col.size, _pd(_f64(U.T).reshape(-1)), K,
                               _pd(y_train), _pd(estim), _pd(std_err)))
    return MHTest(estim, std_err, estim / std_err, n - K - 1)


def univlinreg_last_ms():
    """Device time of the last big_univLinReg call (CUDA events), in ms."""
    return lib().bsg_univlinreg_last_ms()


_GLM_THRESH, _GLM_MTHRESH = 30.0, -30.0  # R's binomial logit: make.link("logit") clamps eta beyond +-30
_DBL_EPS = np.finfo(np.float64).eps


def logit_glm_fit(A, y, eps=1e-8, maxit=25):
    """R's glm.fit for family = binomial() (logit link, unit prior weights) on the design A (no intercept added):
    mustart = (y + 0.5) / 2, iteratively reweighted least squares, converged when |dev - devold| / (|dev| + 0.1) < eps,
    at most maxit iterations.  Returns (coefficients, standard errors from the last weighted fit, iterations, converged)."""
    A, y = _f64(A), _f64(y)

    def linkinv(eta):
        t = np.where(eta < _GLM_MTHRESH, _DBL_EPS, np.where(eta > _GLM_THRESH, 1 / _DBL_EPS, np.exp(eta)))
        return t / (1 + t)

    def mu_eta(eta):
        with np.errstate(over="ignore"):
            e = np.exp(eta)
            return np.where((eta > _GLM_THRESH) | (eta < _GLM_MTHRESH), _DBL_EPS, e / ((1 + e) * (1 + e)))

    def deviance(mu):
        with np.errstate(divide="ignore", invalid="ignore"):
            return 2 * np.sum(np.where(y == 1, -np.log(mu), -np.log1p(-mu)))

    mu = (y + 0.5) / 2
    eta = np.log(mu / (1 - mu))
    devold = deviance(mu)
    coef, Aw, conv, it = np.zeros(A.shape[1]), A, False, 0
    for it in range(1, maxit + 1):
        me = mu_eta(eta)
        z = eta + (y - mu) / me
        w = np.sqrt(me * me / (mu * (1 - mu)))
        Aw = A * w[:, None]
        coef = np.linalg.lstsq(Aw, z * w, rcond=None)[0]
        eta = A @ coef
        mu = linkinv(eta)
        dev = deviance(mu)
        if abs(dev - devold) / (abs(dev) + 0.1) < eps:
            conv = True
            break
        devold = dev
    with np.errstate(invalid="ignore"):
        se = np.sqrt(np.diag(np.linalg.pinv(Aw.T @ Aw)))
    return coef, se, it, conv


def _decode_column(X, ind_train, j):
    """X[ind_train, j] as float64 (column j 1-based): the codes of a hard-call handle, byte / D of a dosage handle."""
    if X.dosage_scale:
        return bed_prodVec(X, np.ones(1), ind_train, _i32([j]))
    return read_bed(X, ind_train, _i32([j]))[:, 0].astype(np.float64)


def big_univLogReg(X, y01_train, ind_train=..., ind_col=..., covar_train=None, tol=1e-8, maxiter=20, ncores=1):
    """bigstatsr's big_univLogReg on the device (bsg_univlogreg): the logistic regression of y01_train on
    [1, covar_train, X[, j]] for every column j of ind_col, by per-SNP IRLS from the null model.  Here in NumPy: the basis
    U of the covariates (univlinreg_covar_basis), the null model glm.fit(U, y01) and, for the SNPs whose IRLS did not meet
    tol in maxiter steps, a glm.fit refit on [U, x] (same span as [1, covar, x], so the same estimate of x).  Returns an
    MHTest with df = None (normal p-values), `niter` and `refitted`."""
    _assert_bed(X)
    ind_train = X.rows_along() if ind_train is ... else _i32(ind_train)
    ind_col = X.cols_along() if ind_col is ... else _i32(ind_col)
    y = _f64(y01_train).reshape(-1)
    _assert_lengths(y, ind_train)
    if not np.all((y == 0) | (y == 1)):
        raise ValueError("'y01.train' should be composed of 0s and 1s.")
    if y.size and (np.all(y == 0) or np.all(y == 1)):
        raise ValueError("'y01.train' should have both 0s and 1s.")
    n = ind_train.size
    if covar_train is not None:
        cv = np.asarray(covar_train, dtype=np.float64)
        if cv.shape[0] != n:
            raise ValueError(ERROR_DIM)
    U = univlinreg_covar_basis(covar_train, n)
    K = U.shape[1]
    gamma0 = logit_glm_fit(U, y)[0]
    m = ind_col.size
    estim, std_err, niter = np.empty(m), np.empty(m), np.empty(m, dtype=np.int32)
    check(lib().bsg_univlogreg(X._h, _pi(ind_train), n, _pi(ind_col), m, _pd(_f64(U.T).reshape(-1)), K, _pd(_f64(gamma0)),
                               _pd(y), float(tol), int(maxiter), _pd(estim), _pd(std_err), _pi(niter)))
    refitted = niter < 0
    niter = np.abs(niter)
    for c in np.flatnonzero(refitted):
        x = _decode_column(X, ind_train, int(ind_col[c]))
        coef, se, it, _ = logit_glm_fit(np.column_stack([U, x]), y)
        estim[c], std_err[c], niter[c] = coef[-1], se[-1], it
    res = MHTest(estim, std_err, estim / std_err, None)
    res.niter, res.refitted = niter, refitted
    return res


def univlogreg_last_ms():
    """Device time of the last big_univLogReg call's IRLS (CUDA events), in ms."""
    return lib().bsg_univlogreg_last_ms()


SPLREG_MESSAGES = ("Complete path", "No more improvement", "Too many variables")


class SpModel:
    """big_spLinReg's / big_spLogReg's result (bigstatsr's `big_sp_list`, power_scale = 1, power_adaptive = 0), one entry
    per alpha, every coefficient on the original scale of the columns:

    - `intercept[A]`, `beta[A][J]` (the kept columns `ind_col`, then the covariates): the mean over the K folds of each
      fold's fit at its best lambda (cross-model selection and averaging);
    - `validation_loss[A]`: the mean over folds of the best validation losses (mean squared error, or mean binomial
      deviance); `nb_var[A]`: nonzero entries of `beta`;
    - `message[A][K]`, `nb_lambda[A][K]` (lambda steps run), `best_lambda[A][K]` (0-based);
    - `path[A][K]`: the whole path of each fit (`lambda`, `loss`, `nnz`, `passes`, and `beta` / `intercept` on the
      standardised scale when the call asked for `return_path`);
    - `center`, `scale`: the column statistics over ind.train of the kept columns then the covariates."""

    def __init__(self, **kw):
        self.__dict__.update(kw)

    def summary(self, best_only=False):
        """One row per alpha (dicts of alpha, intercept, beta, validation_loss, nb_var, message); best_only: the row of
        the alpha with the lowest validation loss."""
        rows = [dict(alpha=float(a), intercept=float(self.intercept[i]), beta=self.beta[i],
                     validation_loss=float(self.validation_loss[i]), nb_var=int(self.nb_var[i]),
                     message=list(self.message[i])) for i, a in enumerate(self.alphas)]
        return rows[self.best_alpha] if best_only else rows

    @property
    def best_alpha(self):
        return int(np.argmin(self.validation_loss))

    def predict(self, X, ind_row=..., covar_row=None, base_row=None):
        """The linear predictor of the best alpha's model at ind_row (also bigstatsr's default for logistic), plus the
        offset base_row when given.  On a Bed the genotype part is bed_prodVec on the device; on a dense float32 /
        float64 matrix (what the model was fitted on) it is X[ind_row, ind_col] @ beta in float64 on the host, one pass
        over the kept columns.  The covariates and the intercept are added on the host.  A missing value on a (row, kept
        column) pair is refused, as in the fit."""
        i = self.best_alpha
        G = self.ind_col.size
        if isinstance(X, Bed):
            ind_row = X.rows_along() if ind_row is ... else _i32(ind_row)
            if G and not X.dosage_scale and bed_counts(X, ind_row, self.ind_col)[3].any():
                raise ValueError("A kept column holds a missing value on 'ind.row'; impute it first "
                                 "(snp_fastImputeSimple).")
            geno = bed_prodVec(X, self.beta[i][:G], ind_row, self.ind_col) if G else np.zeros(ind_row.size)
        else:
            X = _dense_matrix(X)
            ind_row = np.arange(1, X.shape[0] + 1, dtype=np.int32) if ind_row is ... else _i32(ind_row)
            for ind, lim in ((ind_row, X.shape[0]), (self.ind_col, X.shape[1])):
                if ind.size and (ind.min() < 1 or ind.max() > lim):
                    raise IndexError("subscript out of bounds")
            geno = np.zeros(ind_row.size)
            for c0 in range(0, G, 256):  # blocks of kept columns, so that no n x G copy is made
                cols = self.ind_col[c0:c0 + 256] - 1
                geno += X[np.ix_(ind_row - 1, cols)].astype(np.float64) @ self.beta[i][c0:c0 + cols.size]
            if not np.isfinite(geno).all():
                raise ValueError("A kept column holds a non-finite value on 'ind.row'.")
        if np.isnan(geno).any():  # dosage tables: an NA code makes its output NaN
            raise ValueError("A kept column holds a missing value on 'ind.row'; impute it first (snp_fastImputeSimple).")
        out = geno + self.intercept[i]
        if base_row is not None:
            base = _f64(base_row).reshape(-1)
            _assert_lengths(base, ind_row)
            out = out + base
        Kc = self.beta[i].size - G
        if Kc:
            if covar_row is None:
                raise ValueError("'covar.row' is needed: the model has %d covariates." % Kc)
            cv = _f64(covar_row).reshape(ind_row.size, Kc)
            out = out + cv @ self.beta[i][G:]
        return out


def _dense_matrix(X):
    """X as a 2-D float32 / float64 array (an np.memmap or a GridPRS stays what it is); other types: TypeError."""
    X = X if isinstance(X, np.ndarray) else np.asarray(X)
    if X.dtype not in (np.float32, np.float64):
        raise TypeError("A dense matrix must hold float32 or float64 values (not %s)." % X.dtype)
    if X.ndim != 2:
        raise ValueError(ERROR_DIM)
    return X


def _dense_operand(X):
    """(X, dtype code, leading dimension) for bsg_splreg_dense: a column-major matrix (columns may sit ld >= nrow
    elements apart, as in a column slice of a larger one) is passed as it is; any other layout, a C-ordered array
    included, is first copied into a Fortran-ordered one."""
    X = _dense_matrix(X)
    n, it = X.shape[0], X.itemsize
    st0, st1 = X.strides
    if not (X.size == 0 or ((st0 == it or n == 1) and st1 % it == 0 and st1 >= max(n, 1) * it)):
        X = np.asfortranarray(X)
        st1 = max(n, 1) * it
    return X, int(X.dtype == np.float64), (st1 // it if X.size else max(n, 1))


def _big_spreg(family, X, y, ind_train, ind_col, covar_train, base_train, pf_X, pf_covar, alphas, K, ind_sets,
               nlambda, lambda_min_ratio, nlam_min, n_abort, dfmax, eps, max_iter, power_scale, power_adaptive, seed,
               return_path):
    if isinstance(X, Bed):
        nrow, ncol = X.nrow, X.ncol
    else:
        X, dtype, ld = _dense_operand(X)
        nrow, ncol = X.shape
    ind_train = np.arange(1, nrow + 1, dtype=np.int32) if ind_train is ... else _i32(ind_train)
    ind_col = np.arange(1, ncol + 1, dtype=np.int32) if ind_col is ... else _i32(ind_col)
    y = _f64(y).reshape(-1)
    _assert_lengths(y, ind_train)
    nr, nc = ind_train.size, ind_col.size
    Kc = 0
    cov = None
    if covar_train is not None:
        cv = np.asarray(covar_train, dtype=np.float64)
        cv = cv.reshape(-1, 1) if cv.ndim == 1 else cv
        if cv.shape[0] != nr:
            raise ValueError(ERROR_DIM)
        Kc = cv.shape[1]
        cov = _f64(cv.T).reshape(-1)  # column-major
    base = None if base_train is None else _f64(base_train).reshape(-1)
    if base is not None:
        _assert_lengths(base, ind_train)
    pfx = None if pf_X is None else _f64(np.broadcast_to(np.asarray(pf_X, dtype=np.float64), (nc,)))
    pfc = None if pf_covar is None else _f64(np.broadcast_to(np.asarray(pf_covar, dtype=np.float64), (Kc,)))
    alphas = _f64(np.atleast_1d(alphas))
    K = int(K)
    if ind_sets is None:
        ind_sets = (np.random.default_rng(seed).permutation(nr) % K + 1) if K >= 1 else np.ones(nr)
    ind_sets = _i32(ind_sets)
    _assert_lengths(ind_sets, ind_train)
    A, F, Jmax = alphas.size, alphas.size * K, nc + Kc
    center, scale, kept = np.empty(max(Jmax, 1)), np.empty(max(Jmax, 1)), np.zeros(max(nc, 1), dtype=np.uint8)
    beta, b0 = np.zeros(max(F * Jmax, 1)), np.zeros(max(F, 1))
    best, length, msg = (np.zeros(max(F, 1), dtype=np.int32) for _ in range(3))
    lam, loss = np.zeros(max(F * nlambda, 1)), np.zeros(max(F * nlambda, 1))
    nnz, npass = np.zeros(max(F * nlambda, 1), dtype=np.int32), np.zeros(max(F * nlambda, 1), dtype=np.int32)
    pbeta = np.zeros(max(F * nlambda * Jmax, 1)) if return_path else None
    pb0 = np.zeros(max(F * nlambda, 1)) if return_path else None
    tail = (family, _pd(y), _pd(cov), Kc, _pd(base), _pd(pfx), _pd(pfc), _pd(alphas), A, _pi(ind_sets), K, int(nlambda),
            float(lambda_min_ratio), int(nlam_min), int(n_abort), int(dfmax), float(eps), int(max_iter),
            float(power_scale), float(power_adaptive), _pd(center), _pd(scale), kept.ctypes.data_as(_lib.c_u8_p),
            _pd(beta), _pd(b0), _pi(best), _pi(length), _pi(msg), _pd(lam), _pd(loss), _pi(nnz), _pi(npass), _pd(pbeta),
            _pd(pb0))
    if isinstance(X, Bed):
        check(lib().bsg_splreg(X._h, _pi(ind_train), nr, _pi(ind_col), nc, *tail))
    else:
        check(lib().bsg_splreg_dense(C.c_void_p(X.ctypes.data) if X.size else None, dtype, ld, nrow, ncol,
                                     _pi(ind_train), nr, _pi(ind_col), nc, 0, *tail))
    keep = kept[:nc].astype(bool)
    J = int(keep.sum()) + Kc
    cols = np.concatenate([np.flatnonzero(keep), nc + np.arange(Kc)])
    c, s = center[cols], scale[cols]
    beta = beta[:F * J].reshape(A, K, J)
    raw = dict(beta=beta, b0=b0[:F].reshape(A, K), best=best[:F].reshape(A, K), length=length[:F].reshape(A, K),
               message=msg[:F].reshape(A, K))
    ob, oi = splreg_unscale(beta, raw["b0"], c, s)
    path = [[None] * K for _ in range(A)]
    for a in range(A):
        for k in range(K):
            f, L = a * K + k, int(length[a * K + k])
            sl = slice(f * nlambda, f * nlambda + L)
            p = dict(lambda_=lam[sl].copy(), loss=loss[sl].copy(), nnz=nnz[sl].copy(), passes=npass[sl].copy())
            if return_path:
                p["beta"] = pbeta[:F * nlambda * J].reshape(F, nlambda, J)[f, :L].copy()
                p["intercept"] = pb0[sl].copy()
            path[a][k] = p
    best_loss = np.array([[path[a][k]["loss"][raw["best"][a, k]] for k in range(K)] for a in range(A)])
    return SpModel(family="binomial" if family else "gaussian", alphas=alphas, intercept=oi, beta=ob,
                   validation_loss=best_loss.mean(axis=1), nb_var=(ob != 0).sum(axis=1),
                   message=[[SPLREG_MESSAGES[m] for m in raw["message"][a]] for a in range(A)],
                   nb_lambda=raw["length"], best_lambda=raw["best"], path=path, ind_col=ind_col[keep],
                   center=c, scale=s, ind_sets=ind_sets, raw=raw)


def splreg_unscale(beta, b0, center, scale):
    """Cross-model averaging on the original scale: per fit beta_j / s_j and b0 - sum_j c_j beta_j / s_j, then the mean
    over folds.  beta [A][K][J] and b0 [A][K] on the standardised scale."""
    bo = beta / scale
    io = b0 - (bo * center).sum(axis=2)
    return bo.mean(axis=1), io.mean(axis=1)


def big_spLinReg(X, y_train, ind_train=..., ind_col=..., covar_train=None, base_train=None, pf_X=None, pf_covar=None,
                 alphas=1, K=10, ind_sets=None, nlambda=200, lambda_min_ratio=1e-4, nlam_min=50, n_abort=10,
                 dfmax=50000, eps=1e-5, max_iter=1000, power_scale=1, power_adaptive=0, seed=1, return_path=False,
                 ncores=1):
    """bigstatsr's big_spLinReg on the device (bsg_splreg): the elastic net (1/2n)|y - b0 - X beta|^2 +
    lambda sum_j pf_j (alpha |beta_j| + (1 - alpha) / 2 beta_j^2) on standardised columns, K folds x alphas paths with
    early stopping on each fold's held-out loss, averaged over folds (CMSA).  ind_sets fixes the folds; otherwise they
    come from a permutation seeded by `seed` (R's sample is not reproduced).  Returns an SpModel.

    X is a Bed, or a 2-D float32 / float64 matrix (an ndarray, np.memmap or GridPRS; bsg_splreg_dense): X[ind_train,
    ind_col] is read once into device memory in its own type and widened to double exactly when read, so the fit is
    the one of X.astype(float64).  A Fortran-ordered matrix is read in place; a C-ordered one is copied into Fortran
    order first.  Non-finite values on the selected cells are refused."""
    return _big_spreg(0, X, y_train, ind_train, ind_col, covar_train, base_train, pf_X, pf_covar, alphas, K, ind_sets,
                      nlambda, lambda_min_ratio, nlam_min, n_abort, dfmax, eps, max_iter, power_scale, power_adaptive,
                      seed, return_path)


def big_spLogReg(X, y01_train, ind_train=..., ind_col=..., covar_train=None, base_train=None, pf_X=None, pf_covar=None,
                 alphas=1, K=10, ind_sets=None, nlambda=200, lambda_min_ratio=1e-4, nlam_min=50, n_abort=10,
                 dfmax=50000, eps=1e-5, max_iter=1000, power_scale=1, power_adaptive=0, seed=1, return_path=False,
                 ncores=1):
    """bigstatsr's big_spLogReg on the device (bsg_splreg): big_spLinReg's penalty with the mean negative binomial
    log-likelihood as the loss, fitted by coordinate descent on a quadratic approximation whose weights p (1 - p) are
    recomputed at the start of every pass.  y01_train must be 0 / 1.  Returns an SpModel; predict gives the linear
    predictor."""
    return _big_spreg(1, X, y01_train, ind_train, ind_col, covar_train, base_train, pf_X, pf_covar, alphas, K, ind_sets,
                      nlambda, lambda_min_ratio, nlam_min, n_abort, dfmax, eps, max_iter, power_scale, power_adaptive,
                      seed, return_path)


def splreg_last_ms():
    """Device time of the last big_spLinReg / big_spLogReg call (CUDA events), in ms."""
    return lib().bsg_splreg_last_ms()


def splreg_last_stage_ms():
    """Host time of the last big_spLinReg / big_spLogReg call's staging (a dense matrix's gather and upload), in ms."""
    return lib().bsg_splreg_last_stage_ms()


def stacking_fold(w, lpS, grid_lpS_thr, betas, all_keep):
    """R/SCT.R:283-296: per-SNP effects from the stacking weights w (one per column of snp_grid_PRS's matrix).  Keep set
    s (chromosome-major, the order of unlist(all_keep)) owns columns s n_thr .. (s + 1) n_thr - 1; each of its SNPs gets
    c(0, cumsum(b))[1 + sum(lp > grid_lpS_thr)] of that set's weights b (cumsum in long double, as R's), added over the
    sets that hold it; beta.G = coef * betas.  A NaN lpS inside a set gives a NaN coefficient (R's NA index); SNPs in
    no set get 0 * beta (NaN for a NaN beta)."""
    thr = np.asarray(grid_lpS_thr, dtype=np.float64).reshape(-1)
    lpS, betas, w = (np.asarray(v, dtype=np.float64).reshape(-1) for v in (lpS, betas, w))
    nthr = thr.size
    coef = np.zeros(betas.size)
    s = 0
    for chrom in all_keep:
        for keep in chrom:
            keep = np.asarray(keep, dtype=np.int64).reshape(-1) - 1
            b2 = np.concatenate([[0.0], np.cumsum(w[s:s + nthr].astype(np.longdouble)).astype(np.float64)])
            lp = lpS[keep]
            add = b2[(lp[:, None] > thr).sum(axis=1)]
            add[np.isnan(lp)] = np.nan
            coef[keep] = coef[keep] + add
            s += nthr
    if s != w.size:
        raise ValueError("'multi_PRS' has %d columns; its keep sets and thresholds make %d." % (w.size, s))
    return coef * betas


def snp_grid_stacking(multi_PRS, y_train, alphas=(1, 0.01, 0.0001), ncores=1, **kw):
    """R/SCT.R:266-304: stacking over snp_grid_PRS's C+T scores.  big_spLogReg when y_train has exactly two distinct
    values (they must be 0 / 1), big_spLinReg otherwise, over the dense score matrix on the device (**kw forwarded:
    K, covar_train, pf_covar, ind_train, ind_col, ind_sets, seed, ...); then the best alpha's weights of the kept
    columns are folded into per-SNP effects (stacking_fold).  Returns R's list: `intercept`, `beta.G`, `beta.covar`,
    `mod` (the SpModel)."""
    attrs = [getattr(multi_PRS, a, None) for a in ("lpS", "grid_lpS_thr", "betas", "all_keep")]
    if any(a is None for a in attrs):
        raise ValueError("'multi_PRS' must be the result of snp_grid_PRS (attributes lpS, grid_lpS_thr, betas, "
                         "all_keep).")
    lpS, thr, betas, all_keep = attrs
    y = _f64(y_train).reshape(-1)
    fit = big_spLogReg if np.unique(y).size == 2 else big_spLinReg
    mod = fit(multi_PRS, y, alphas=alphas, ncores=ncores, **kw)
    best = mod.summary(best_only=True)
    G = mod.ind_col.size
    w = np.zeros(multi_PRS.shape[1])
    w[mod.ind_col - 1] = best["beta"][:G]
    return {"intercept": best["intercept"], "beta.G": stacking_fold(w, lpS, thr, betas, all_keep),
            "beta.covar": best["beta"][G:], "mod": mod}
