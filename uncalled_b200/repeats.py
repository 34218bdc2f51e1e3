"""`find-repeats`: how long the sequence starting at each reference position stays repeated in the reference (the
reference's `src/find_repeats.cpp`, on the GPU).

The repeat length L(p) of a position is the number of FM-index steps of `self_align`'s walk from p
(src/self_align_ref.cpp:64-84): the search follows the contig forward from p with complemented bases until the range
holds at most one row or the contig ends.  So the L + 1 bases from p occur at most once in the reference and its
reverse complement (bwa's concatenated text, so across contig ends too), or p + L is the contig's last base.  A read
from a stretch repeated for longer than a seed cannot be placed by the mapper.

    f = RepeatFinder("ref")              # ref.bwt / .sa / .pac / .ann / .amb
    f.lengths("chr1", 10000, 20000)      # np.uint32 L for positions [10000, 20000) of chr1
    for L, name, p in f.records(30): ...

Positions inside an `.amb` hole (a run of N in the FASTA) have random `.pac` bases: `records` skips them and the
sequences it reports print their bases as N; `lengths` returns their raw walk values."""
import ctypes as C
import os

import numpy as np

from . import _native as N

WINDOW = 1 << 24        # positions per device call: 64 MB of lengths on the device and on the host
EXTS = (".bwt", ".sa", ".pac", ".ann", ".amb")


class IndexFileError(ValueError):
    """a missing or inconsistent index file, found before the GPU is touched"""


def read_layout(prefix):
    """(contigs [(name, .pac offset, length)], hole starts, hole ends (.pac positions, sorted), l_pac) of a bwa index,
    after checking that its files exist and agree with each other"""
    for e in EXTS:
        if not os.path.isfile(prefix + e):
            raise IndexFileError("'%s' does not exist" % (prefix + e))
    try:
        with open(prefix + ".ann") as f:
            l_pac, n_seqs = (int(v) for v in f.readline().split()[:2])
            contigs = []
            for _ in range(n_seqs):
                name = f.readline().split()[1]
                off, ln = (int(v) for v in f.readline().split()[:2])
                contigs.append((name, off, ln))
        with open(prefix + ".amb") as f:
            a_pac, a_seqs, n_holes = (int(v) for v in f.readline().split()[:3])
            holes = np.array([[int(v) for v in f.readline().split()[:2]] for _ in range(n_holes)], np.int64).reshape(-1, 2)
    except (ValueError, IndexError) as e:
        raise IndexFileError("cannot parse the .ann / .amb of %s: %s" % (prefix, e))
    st = 0
    for name, off, ln in contigs:
        if off != st or ln < 0:
            raise IndexFileError("%s.ann: contig %s does not follow the one before it" % (prefix, name))
        st += ln
    if st != l_pac or not contigs or l_pac == 0:
        raise IndexFileError("%s.ann: the contig lengths do not add up to its reference length %d" % (prefix, l_pac))
    if (a_pac, a_seqs) != (l_pac, len(contigs)):
        raise IndexFileError("%s.amb does not describe the reference of %s.ann" % (prefix, prefix))
    if os.path.getsize(prefix + ".pac") < (l_pac + 3) // 4:
        raise IndexFileError("%s.pac is shorter than the reference" % prefix)
    head = np.fromfile(prefix + ".bwt", np.uint64, 5)
    if len(head) < 5 or int(head[4]) != 2 * l_pac:
        raise IndexFileError("%s.bwt does not index the reference of %s.ann" % (prefix, prefix))
    holes = holes[np.argsort(holes[:, 0], kind="stable")]
    return contigs, holes[:, 0], holes[:, 0] + holes[:, 1], l_pac


def check_min_k(min_k):
    if isinstance(min_k, bool) or not isinstance(min_k, (int, np.integer)) or min_k < 0:
        raise ValueError("min_k must be a non-negative integer")


def merge_intervals(st, en):
    """the union of intervals [st, en) given sorted by st, as sorted disjoint intervals; overlapping and book-ended
    ones are joined"""
    st, en = np.asarray(st, np.int64), np.asarray(en, np.int64)
    if not len(st):
        return st, en
    run_en = np.maximum.accumulate(en)
    first = np.flatnonzero(np.concatenate([[True], st[1:] > run_en[:-1]]))
    return st[first], run_en[np.append(first[1:] - 1, len(st) - 1)]


class RepeatFinder:
    """The repeat length of every position of a bwa index's reference, computed on the GPU (`unc_repeats_*`).  The
    index and the packed reference stay on the device until `close`."""

    def __init__(self, bwa_prefix, device=0, window=WINDOW):
        self.prefix = bwa_prefix
        contigs, self._hole_st, self._hole_en, self.l_pac = read_layout(bwa_prefix)
        self.contigs = [(name, ln) for name, _, ln in contigs]
        self._off = {name: (off, ln) for name, off, ln in contigs}
        self.window = int(window)
        self._L = N.lib()
        self._h = C.c_void_p()
        N.check(self._L.unc_init(int(device)))
        N.check(self._L.unc_repeats_create(os.fsencode(bwa_prefix), C.byref(self._h)))

    def close(self):
        if getattr(self, "_h", None):
            self._L.unc_repeats_destroy(self._h)
            self._h = None

    __del__ = close

    def __enter__(self):
        return self

    def __exit__(self, *a):
        self.close()

    def _raw(self, pac_st, n):
        out = np.empty(n, np.uint32)
        for o in range(0, n, self.window):
            k = min(self.window, n - o)
            N.check(self._L.unc_repeats_lengths(self._h, pac_st + o, k, out[o:].ctypes.data))
        return out

    def _contig(self, name):
        if name not in self._off:
            raise KeyError("no contig %r in %s.ann" % (name, self.prefix))
        return self._off[name]

    def lengths(self, name, st=0, en=None):
        """L of positions [st, en) of contig `name` as np.uint32 (hole positions included, as raw walk values)"""
        off, ln = self._contig(name)
        en = ln if en is None else en
        if not 0 <= st <= en <= ln:
            raise ValueError("positions [%d, %d) are not within contig %s of length %d" % (st, en, name, ln))
        return self._raw(off + st, en - st)

    def in_hole(self, pac_pos):
        """whether each .pac position lies in an .amb hole"""
        q = np.asarray(pac_pos, np.int64)
        if not len(self._hole_st):
            return np.zeros(q.shape, bool)
        i = np.searchsorted(self._hole_st, q, side="right") - 1
        return (i >= 0) & (q < self._hole_en[np.maximum(i, 0)])

    def reported(self, min_k):
        """(name, positions, lengths) per window, in .ann order then position order: the positions outside the holes
        whose L >= min_k"""
        check_min_k(min_k)
        return self._reported(min_k)

    def _reported(self, min_k):
        for name, ln in self.contigs:
            off = self._off[name][0]
            for w in range(0, ln, self.window):
                n = min(self.window, ln - w)
                L = self._raw(off + w, n)
                keep = (L >= min_k) & ~self.in_hole(np.arange(off + w, off + w + n))
                p = np.flatnonzero(keep)
                yield name, p + w, L[p]

    def records(self, min_k):
        """(L, contig name, position) of every reported position: L >= min_k and not in an .amb hole"""
        windows = self.reported(min_k)
        return ((li, name, pi) for name, p, L in windows for pi, li in zip(p.tolist(), L.tolist()))

    def bases(self, name):
        """the contig's forward bases as A/C/G/T bytes, with the bases of .amb holes as N"""
        off, ln = self._contig(name)
        b0 = off // 4
        pac = np.fromfile(self.prefix + ".pac", np.uint8, count=(off + ln + 3) // 4 - b0, offset=b0)
        codes = np.empty(pac.size * 4, np.uint8)
        for k in range(4):
            codes[k::4] = (pac >> (6 - 2 * k)) & 3
        codes = codes[off - 4 * b0:off - 4 * b0 + ln]
        h = (self._hole_en > off) & (self._hole_st < off + ln)
        for s, e in zip(self._hole_st[h].tolist(), self._hole_en[h].tolist()):
            codes[max(s - off, 0):min(e - off, ln)] = 4
        return np.frombuffer(b"ACGTN", np.uint8)[codes].tobytes()


def write_lines(finder, min_k, out):
    """find_repeats.cpp's output (src/find_repeats.cpp:77-81): `L contig p p+L seq` per reported position"""
    cur, seq = None, b""
    for name, p, L in finder.reported(min_k):
        if name != cur:
            cur, seq = name, finder.bases(name).decode()
        out.write("".join("%d\t%s\t%d\t%d\t%s\n" % (li, name, pi, pi + li, seq[pi:pi + li])
                          for pi, li in zip(p.tolist(), L.tolist())))


def write_bed(finder, min_k, out):
    """BED of the union of [p, p + L) over the reported positions, per contig, merged and sorted"""
    cur, carry = None, None

    def flush():
        if carry is not None:
            out.write("%s\t%d\t%d\n" % (cur, carry[0], carry[1]))

    for name, p, L in finder.reported(min_k):
        if name != cur:
            flush()
            cur, carry = name, None
        nz = L > 0
        st, en = p[nz].astype(np.int64), p[nz] + L[nz].astype(np.int64)
        if carry is not None:                      # the last run so far starts before every position of this window
            st, en = np.concatenate([[carry[0]], st]), np.concatenate([[carry[1]], en])
        st, en = merge_intervals(st, en)
        if not len(st):
            continue
        out.write("".join("%s\t%d\t%d\n" % (name, s, e) for s, e in zip(st[:-1].tolist(), en[:-1].tolist())))
        carry = (int(st[-1]), int(en[-1]))
    flush()
