"""A functional stand-in for the ``portion`` package (not installed here), written from its documented semantics, so that
the reference's detect_break_points / break_and_update_ctgs can run unmodified when the correction goldens are made.

Covers what HapHiC_cluster.py uses: ``closed(a, b)``, ``empty()``, ``|`` (union; closed intervals that touch merge),
``-`` (difference), ``len()`` (number of atomic intervals), iteration (atomic intervals), ``.lower`` / ``.upper`` and
``overlaps``.  An interval is a sorted list of disjoint atomic intervals (lower, lower_closed, upper, upper_closed)."""


class Interval:
    def __init__(self, atoms=()):
        self._atoms = _normalise(list(atoms))

    @property
    def lower(self):
        return self._atoms[0][0] if self._atoms else float("inf")

    @property
    def upper(self):
        return self._atoms[-1][2] if self._atoms else float("-inf")

    @property
    def empty(self):
        return not self._atoms

    def __len__(self):
        return len(self._atoms)

    def __iter__(self):
        return (Interval([a]) for a in self._atoms)

    def __or__(self, other):
        return Interval(self._atoms + other._atoms)

    def __sub__(self, other):
        out = []
        for a in self._atoms:
            pieces = [a]
            for b in other._atoms:
                nxt = []
                for p in pieces:
                    nxt += _atom_minus(p, b)
                pieces = nxt
            out += pieces
        return Interval(out)

    def overlaps(self, other):
        return any(_atoms_intersect(a, b) for a in self._atoms for b in other._atoms)

    def __eq__(self, other):
        return isinstance(other, Interval) and self._atoms == other._atoms

    def __repr__(self):
        if not self._atoms:
            return "()"
        return " | ".join("{}{},{}{}".format("[" if lc else "(", lo, hi, "]" if hc else ")") for lo, lc, hi, hc in self._atoms)


def _is_empty(a):
    lo, lc, hi, hc = a
    return lo > hi or (lo == hi and not (lc and hc))


def _atoms_intersect(a, b):
    lo, lc = max((a[0], not a[1]), (b[0], not b[1]))      # the larger lower bound (open beats closed at equal values)
    hi, hc = min((a[2], a[3]), (b[2], b[3]))              # the smaller upper bound (open beats closed at equal values)
    return not _is_empty((lo, not lc, hi, hc))


def _normalise(atoms):
    atoms = sorted((a for a in atoms if not _is_empty(a)), key=lambda a: (a[0], not a[1]))
    out = []
    for a in atoms:
        if out:
            p = out[-1]
            # merge when they overlap or touch with at least one closed end at the shared value
            if a[0] < p[2] or (a[0] == p[2] and (a[1] or p[3])):
                if (a[2], a[3]) > (p[2], p[3]):
                    out[-1] = (p[0], p[1], a[2], a[3])
                continue
        out.append(a)
    return out


def _atom_minus(a, b):
    if not _atoms_intersect(a, b):
        return [a]
    res = []
    left = (a[0], a[1], b[0], not b[1])
    right = (b[2], not b[3], a[2], a[3])
    for p in (left, right):
        if not _is_empty(p) and _atoms_intersect(p, a):
            lo = max((a[0], not a[1]), (p[0], not p[1]))
            hi = min((a[2], a[3]), (p[2], p[3]))
            q = (lo[0], not lo[1], hi[0], hi[1])
            if not _is_empty(q):
                res.append(q)
    return res


def closed(lower, upper):
    return Interval([(lower, True, upper, True)])


def empty():
    return Interval()
