"""Test-only: the edge table of the feature-mix kernels (csrc/featmix.cuh, DESIGN.md §3.1m), a second oracle that runs lhotse's
own mixer on it in float64, and the NaN-aware gate shared by tests/test_featmix_kernel_edges.py.

A table is a list of `Cut`s, each a list of `Track`s that state everything the planner (lhotse_b200/precomputed.py) would
write for them: the rows or a constant, the duplicated last row, the offset, the SNR, the flags and the reference.  `build`
lays them out as the planner does (audible tracks in order, a muted reference last with only the ENERGY flag, a zero-row
reference in its place with only the ENERGY flag) and checks that it can.  `lhotse_mix` is not derived from the kernel: it
calls lhotse's `_scale_features_for_snr`, `FeatureMixer.add_to_mix` and `mixed_feats` on float64 rows, then
`MixedCut.load_features`' one-row trim or repeat."""
import math
import zlib
from dataclasses import dataclass
from typing import Optional, Tuple, Union

import numpy as np

import featmix_cases as FC

LOG, LINEAR, COPY, MIX = FC.LOG, FC.LINEAR, FC.COPY, FC.MIX
M, E, ME = FC.MIXED, FC.ENERGY, FC.MIXED | FC.ENERGY
FRAME_SHIFT, SR = 0.01, 16000         # offsets in seconds are off * 0.01 at 16 kHz: compute_num_frames gives off back
PAD = -23.025850929940457             # LOG_EPSILON, the batch's padding value
LOG_EPS = math.log(FC.EPSILON)        # what a log-law element is where the EPSILON clamp binds
F = 5


@dataclass(frozen=True)
class Const:
    """A PaddingCut track: `num_rows` rows of float32 `value`."""
    value: float
    num_rows: int


@dataclass(frozen=True)
class Track:
    x: Union[np.ndarray, Const]   # the stored float32 rows (stored, F), or a constant
    dup: bool                     # the last stored row once more (MonoCut.load_features one row short)
    offset: int                   # in frames
    snr: Optional[float]          # dB; the planner's factor is 10 ** (-snr / 10)
    flags: int                    # MIXED and / or ENERGY
    ref: bool                     # the SNR reference

    @property
    def num_rows(self):
        return self.x.num_rows if isinstance(self.x, Const) else len(self.x) + int(self.dup)

    def rows64(self):
        """The (num_rows, F) float64 rows lhotse loads for the track."""
        if isinstance(self.x, Const):
            return np.full((self.x.num_rows, F), np.float64(np.float32(self.x.value)))
        r = self.x.astype(np.float64)
        return np.concatenate([r, r[-1:]]) if self.dup else r


@dataclass(frozen=True)
class Cut:
    name: str
    mode: int              # COPY or MIX
    law: int               # LOG or LINEAR (a COPY cut states LOG, which it ignores)
    tracks: Tuple[Track, ...]
    adjust: int            # MIX: num_rows - mix_rows (-1 trimmed, 0, +1 the last row repeated); COPY: rows of padding
    pad_value: float       # COPY: the PaddingCut's feat_value after the rows; MIX cuts state 0.0, which they ignore

    def mix_rows(self):
        if self.mode == COPY:
            return 0
        rows = self.tracks[0].num_rows
        for t in self.tracks[1:]:
            if t.flags & M:
                rows = max(rows, t.offset + t.num_rows)
        return rows

    def num_rows(self):
        return self.tracks[0].num_rows + self.adjust if self.mode == COPY else self.mix_rows() + self.adjust

    def ref_k(self):
        return next(k for k, t in enumerate(self.tracks) if t.ref)


@dataclass
class Table:
    cuts: list
    src: np.ndarray
    tracks: np.ndarray
    table: np.ndarray
    T: int


def build(cuts, T=None) -> Table:
    """The kernel tables of `cuts`, after checking that they are laid out as precomputed.py lays them out."""
    from lhotse_b200.engine import FEATMIX_CUT_DTYPE, FEATMIX_TRACK_DTYPE

    src, tracks, table = [], [], []
    elem = 0
    for c, cut in enumerate(cuts):
        tr = cut.tracks
        assert tr[0].flags & M and tr[0].offset == 0, cut.name
        if cut.mode == COPY:
            assert len(tr) == 1 and tr[0].snr is None and cut.adjust >= 0, cut.name
        else:
            assert sum(t.ref for t in tr) == 1 and tr[cut.ref_k()].flags & E, cut.name
            assert tr[0].flags == (ME if tr[0].ref or tr[0].snr is not None else M), cut.name
            for k, t in enumerate(tr):
                assert t.flags in (M, ME, E), cut.name
                if t.snr is not None and (k > 0 or not tr[0].ref):
                    assert t.flags & E, (cut.name, k, "a track with an SNR gives its energy")
                if t.flags == E:  # only a reference gives energy without being mixed: muted (last) or zero-row (in place)
                    assert t.ref and (k == len(tr) - 1 or t.num_rows == 0), (cut.name, k)
                elif k > 0:
                    assert t.num_rows > 0 and not (t.flags & E and t.snr is None and not t.ref), (cut.name, k)
            assert abs(cut.adjust) <= 1 and cut.num_rows() >= 1, cut.name
        first = len(tracks)
        for t in tr:
            stored = 0 if isinstance(t.x, Const) else len(t.x)
            assert isinstance(t.x, Const) and not t.dup or not isinstance(t.x, Const) and t.x.dtype == np.float32 and \
                t.x.shape[1:] == (F,) and (stored > 0 or not t.dup), (cut.name, t)
            if stored:
                pad = (-elem) % 4
                src.append(np.zeros(pad, np.float32))
                elem += pad
                src.append(t.x.ravel())
            factor = math.nan if t.snr is None else 10.0 ** (-t.snr / 10)
            value = float(np.float32(t.x.value)) if isinstance(t.x, Const) else 0.0
            tracks.append((FEATMIX_TRACK_DTYPE.itemsize, c, t.flags, stored, t.num_rows, t.offset, value, 0, elem, factor))
            elem += stored * F
        table.append((FEATMIX_CUT_DTYPE.itemsize, cut.mode, cut.law, cut.num_rows(), cut.mix_rows(), first, len(tr),
                      0 if cut.mode == COPY else cut.ref_k(), np.float32(cut.pad_value), 0))
    table = np.array(table, dtype=FEATMIX_CUT_DTYPE)
    T = int(table["num_rows"].max()) + 1 if T is None else T
    return Table(list(cuts), np.concatenate(src) if src else np.zeros(0, np.float32),
                 np.array(tracks, dtype=FEATMIX_TRACK_DTYPE), table, T)


def evaluate(tab: Table):
    return FC.evaluate(tab.src, tab.tracks, tab.table, F, tab.T, PAD)


# ---- lhotse's own mixer ---------------------------------------------------------------------------------------------------

def _lhotse():
    import pytest

    import refshim

    if not refshim.reference_available():
        pytest.skip("lhotse (oracle/_ref/lhotse_ref.zip) not present")
    refshim.import_reference()  # lhotse's mixer only: lhotse_b200's classes are not re-bound


def lhotse_mix(tab: Table):
    """(B, T, F) float64: each MIX cut through lhotse's `_scale_features_for_snr`, `FeatureMixer(reference_energy=...)`,
    `add_to_mix` (offsets in seconds) and `mixed_feats` on float64 rows, then trimmed or repeated by a row; each COPY cut
    through `MixedCut.load_features`' padding-only branch.  The statics are lhotse's Fbank (log law) and Spectrogram
    (linear law).  Skips without the reference."""
    _lhotse()
    from lhotse.cut.mixed import _scale_features_for_snr
    from lhotse.features.kaldi.extractors import Fbank, Spectrogram
    from lhotse.features.mixer import FeatureMixer

    out = np.full((len(tab.cuts), tab.T, F), np.float64(np.float32(PAD)))
    with np.errstate(all="ignore"):
        for c, cut in enumerate(tab.cuts):
            first = cut.tracks[0]
            if cut.mode == COPY:
                feats = np.ones((cut.num_rows(), F)) * float(np.float32(cut.pad_value))
                feats[: first.num_rows] = first.rows64()
                out[c, : cut.num_rows()] = feats
                continue
            ex = Fbank if cut.law == LOG else Spectrogram
            ref = cut.tracks[cut.ref_k()]
            reference_energy = None if ref is first else ex.compute_energy(ref.rows64())
            base = _scale_features_for_snr(first.rows64(), feature_extractor=ex, snr=first.snr,
                                           reference_energy=reference_energy)
            mixer = FeatureMixer(feature_extractor=ex, base_feats=base, frame_shift=FRAME_SHIFT, reference_energy=reference_energy)
            for t in cut.tracks[1:]:
                if t.flags & M:
                    mixer.add_to_mix(feats=t.rows64(), sampling_rate=SR, snr=t.snr, offset=t.offset * FRAME_SHIFT)
            feats = mixer.mixed_feats
            n = cut.num_rows()
            if feats.shape[0] - n == 1:
                feats = feats[:n]
            if feats.shape[0] - n == -1:
                feats = np.concatenate((feats, feats[-1:]), axis=0)
            assert feats.shape == (n, F), cut.name
            out[c, :n] = feats
    return out


# ---- the gates ------------------------------------------------------------------------------------------------------------

def nan_gate(got, truth, bound, what=""):
    """NaN exactly where the truth is NaN, +-inf exactly where it is +-inf, |got - truth| <= bound on the finite rest."""
    got, truth = np.asarray(got, np.float64), np.asarray(truth, np.float64)
    assert got.shape == truth.shape, (what, got.shape, truth.shape)
    bound = np.broadcast_to(np.asarray(bound, np.float64), truth.shape)

    def first(mask, why):
        i = tuple(int(v[0]) for v in np.nonzero(mask))
        return f"{what}: {int(mask.sum())} elements {why}, first at {i}: got {got[i]!r}, want {truth[i]!r}"

    nan = np.isnan(truth)
    assert np.array_equal(np.isnan(got), nan), first(np.isnan(got) != nan, "with NaN in one and not the other")
    inf = np.isinf(truth)
    assert (got[inf] == truth[inf]).all(), first(inf & (got != truth), "where the truth is infinite")
    fin = np.isfinite(truth)
    with np.errstate(invalid="ignore"):
        bad = fin & ~(np.abs(got - truth) <= bound)
    assert not bad.any(), first(bad, "over the bound")


def ulp_gate(got, truth, what=""):
    """The hand-table gate: ulp32(truth) on the finite elements."""
    with np.errstate(all="ignore"):
        nan_gate(got, truth, FC.ulp32(np.where(np.isfinite(truth), truth, 0.0)), what)


def cut_gate(ours, lhotse32, truth64, what=""):
    """The strategy gate: per cut 2 E_cut + ulp32(truth), E_cut the largest |lhotse - truth| over the elements where both are
    finite."""
    ours, lhotse32, truth64 = (np.asarray(a, np.float64) for a in (ours, lhotse32, truth64))
    assert ours.shape == lhotse32.shape == truth64.shape
    for c in range(ours.shape[0]):
        both = np.isfinite(lhotse32[c]) & np.isfinite(truth64[c])
        e_cut = float(np.max(np.abs(lhotse32[c][both] - truth64[c][both]))) if both.any() else 0.0
        with np.errstate(all="ignore"):
            bound = 2 * e_cut + FC.ulp32(np.where(np.isfinite(truth64[c]), truth64[c], 0.0))
        nan_gate(ours[c], truth64[c], bound, f"{what} cut {c}")


def copy_bits_equal(got, want):
    """Bit for bit (so -0.0 stays -0.0), NaN positions equal (their payloads are not compared)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    nan = np.isnan(want)
    return np.array_equal(np.isnan(got), nan) and np.array_equal(got.view(np.int32)[~nan], want.view(np.int32)[~nan])


# ---- the table ------------------------------------------------------------------------------------------------------------

def _rs(*key):
    return np.random.RandomState(zlib.crc32(repr(key).encode()))


def pos(rs, law, n):
    """Rows of positive energy: log-mel-like (log law) or power-like (linear law)."""
    x = rs.randn(n, F)
    return (x * 2 - 5 if law == LOG else np.abs(x) + 0.05).astype(np.float32)


def neg(rs, law, n):
    """Rows of zero energy: all -inf (log law, e^-inf = 0) or non-positive with a negative sum (linear law)."""
    return np.full((n, F), -np.inf, np.float32) if law == LOG else (-np.abs(rs.randn(n, F)) - 0.05).astype(np.float32)


def near_eps(rs, law, n):
    """Log law: values from -23.6 to -22.4 in steps of 0.1, so that e^x falls on both sides of EPSILON and no element is within
    1e-3 of log(EPSILON); the linear law takes `pos` rows."""
    if law == LINEAR:
        return pos(rs, law, n)
    grid = np.round(np.arange(-23.6, -22.35, 0.1), 1)
    return rs.choice(grid, size=(n, F)).astype(np.float32)


def put(x, *cells):
    """A copy of `x` with (row, col, value) cells set."""
    x = x.copy()
    for r, c, v in cells:
        x[r, c] = v
    return x


NAN, INF = np.float32(np.nan), np.float32(np.inf)
EMPTY = np.zeros((0, F), np.float32)


def tr(x, dup, off, snr, flags, ref):
    return Track(x, dup, off, snr, flags, ref)


def mix(name, law, tracks, adjust):
    return Cut(f"{name}/{'log' if law == LOG else 'linear'}", MIX, law, tuple(tracks), adjust, 0.0)


def edge_cuts():
    """Every row of the edge table, each MIX row under both laws."""
    cuts = []
    for law in (LOG, LINEAR):
        def rs(name):
            return _rs(name, law)

        def p(name, n):
            return pos(rs(name), law, n)

        # the reference: track 0, a later mixed track without or with its own SNR, a muted track, a zero-row track
        cuts += [
            mix("ref_first", law, [tr(p("rf0", 4), False, 0, None, ME, True), tr(p("rf1", 3), False, 2, 10.0, ME, False)], 0),
            mix("ref_later_no_snr", law, [tr(p("rl0", 4), False, 0, 5.0, ME, False), tr(p("rl1", 5), False, 1, None, ME, True),
                                          tr(p("rl2", 2), False, 3, -3.0, ME, False)], -1),
            mix("ref_later_own_snr", law, [tr(p("rs0", 3), False, 0, 3.0, ME, False), tr(p("rs1", 3), True, 0, 7.0, ME, True)], 1),
            mix("ref_muted", law, [tr(p("rm0", 4), False, 0, 2.0, ME, False), tr(p("rm1", 2), False, 1, 12.0, ME, False),
                                   tr(p("rm2", 6), False, 0, None, E, True)], 0),
            mix("ref_zero_rows", law, [tr(p("rz0", 3), False, 0, 4.0, ME, False), tr(EMPTY, False, 0, None, E, True),
                                       tr(p("rz2", 2), False, 1, 6.0, ME, False),
                                       tr(Const(-4.5 if law == LOG else 0.25, 2), False, 3, None, M, False)], 0),
        ]
        # the first track's scaling when the reference is another track
        cuts += [
            mix("first_e_ref_le0", law, [tr(p("e00", 4), False, 0, 6.0, ME, False), tr(p("e01", 2), False, 2, 3.0, ME, False),
                                         tr(neg(rs("e02"), law, 3), False, 0, None, E, True)], 0),
            mix("first_e0_le0", law, [tr(neg(rs("e10"), law, 4), False, 0, 6.0, ME, False),
                                      tr(p("e11", 3), False, 1, None, ME, True)], 0),
            mix("first_e_ref_nan", law, [tr(p("e20", 4), False, 0, 6.0, ME, False),
                                         tr(put(p("e21", 3), (1, 2, NAN)), False, 1, None, ME, True)], 0),
            mix("first_e0_nan", law, [tr(put(p("e30", 4), (2, 1, NAN)), False, 0, 6.0, ME, False),
                                      tr(p("e31", 3), False, 1, None, ME, True)], 0),
            mix("first_e0_inf", law, [tr(put(p("e40", 4), (0, 3, INF)), False, 0, 6.0, ME, False),
                                      tr(p("e41", 3), False, 1, None, ME, True)], 0),
            mix("first_gain_inf", law, [tr(p("e50", 3), False, 0, 6.0, ME, False), tr(p("e51", 2), False, 1, None, M, False),
                                        tr(put(p("e52", 2), (1, 4, INF)), False, 0, None, E, True)], 0),
        ]
        # a MIX cut that mixes nothing into its (scaled) first track: fm_output's `added == false`
        cuts += [
            mix("not_added_muted_ref", law, [tr(p("na0", 4), True, 0, 6.0, ME, False), tr(p("na1", 3), False, 0, None, E, True)], 0),
            mix("not_added_zero_ref", law, [tr(p("nz0", 3), False, 0, -4.0, ME, False), tr(EMPTY, False, 0, None, E, True)], -1),
        ]
        # the EPSILON clamp on some elements only: gaps, a track past the base's end, a track at mix_rows - 1, values near -23.03
        cuts += [
            mix("gap_past_base_end", law, [tr(near_eps(rs("g0"), law, 3), False, 0, None, ME, True),
                                           tr(p("g1", 2), False, 5, 10.0, ME, False), tr(p("g2", 1), False, 6, 20.0, ME, False)], -1),
            mix("last_row_offset", law, [tr(near_eps(rs("l0"), law, 4), True, 0, None, ME, True),
                                         tr(near_eps(rs("l1"), law, 1), False, 3, None, M, False),
                                         tr(p("l2", 1), False, 4, 30.0, ME, False)], 1),
            mix("near_eps_both_sides", law, [tr(near_eps(rs("n0"), law, 5), False, 0, None, ME, True),
                                              tr(near_eps(rs("n1"), law, 3), False, 1, None, M, False)], 0),
        ]
        # NaN, +inf and -inf in a base row, inside a further track's window, in the reference's rows
        cuts += [
            mix("nonfinite_base", law, [tr(put(p("b0", 4), (1, 2, NAN), (2, 0, INF), (0, 4, -INF), (3, 1, -INF)), False, 0, None, M,
                                           False), tr(p("b1", 2), False, 1, 5.0, ME, False), tr(p("b2", 4), False, 0, None, E, True)], 0),
            mix("nonfinite_base_is_ref", law, [tr(put(p("bb0", 3), (1, 3, NAN)), False, 0, None, ME, True),
                                               tr(p("bb1", 2), False, 1, 8.0, ME, False)], 0),
            mix("nonfinite_further", law, [tr(p("f0", 4), False, 0, None, ME, True),
                                           tr(put(p("f1", 3), (0, 1, NAN), (1, 3, -INF)), False, 1, 5.0, ME, False),
                                           tr(put(p("f2", 2), (0, 0, INF)), False, 2, None, M, False),
                                           tr(put(p("f3", 2), (1, 2, INF)), False, 0, 10.0, ME, False)], 0),
            mix("nonfinite_ref_pos_inf", law, [tr(p("r0", 3), False, 0, 6.0, ME, False),
                                               tr(put(p("r1", 2), (0, 2, INF)), False, 1, None, ME, True),
                                               tr(p("r2", 2), False, 0, 3.0, ME, False)], 0),
            mix("nonfinite_ref_neg_inf", law, [tr(p("q0", 3), False, 0, 6.0, ME, False),
                                               tr(put(p("q1", 2), (1, 1, -INF)), False, 0, None, ME, True),
                                               tr(p("q2", 2), False, 1, 3.0, ME, False)], 0),
        ]
    # COPY cuts keep their rows bit for bit: NaN, +-inf, -0.0, a repeated last row, the padding value after them
    rs = _rs("copy")
    x = put(pos(rs, LOG, 4), (0, 0, NAN), (1, 1, INF), (2, 2, -INF), (3, 3, np.float32(-0.0)), (0, 4, np.float32(-0.0)))
    cuts += [Cut("copy_nonfinite", COPY, LOG, (tr(x, False, 0, None, M, False),), 2, -9.5),
             Cut("copy_dup_negzero_pad", COPY, LOG, (tr(put(pos(rs, LINEAR, 2), (1, 0, NAN)), True, 0, None, M, False),), 1, -0.0),
             Cut("copy_exact", COPY, LOG, (tr(put(pos(rs, LOG, 3), (2, 1, -INF)), False, 0, None, M, False),), 0, 7.0)]
    return cuts


def batch_cuts(n):
    """`n` one-row cuts cycling through a log-law mix with the reference first, a linear-law mix whose scaled first track is
    all there is, a log-law mix trimmed to one row, and a copy; every cut's rows its own."""
    rs = _rs("batch", n)
    x = rs.randn(n, 2, F).astype(np.float32)
    cuts = []
    for c in range(n):
        a, b = x[c, :1], x[c, 1:]
        kind = c % 4
        if kind == 0:
            cuts.append(Cut(f"b{c}", MIX, LOG, (tr(a - 4, False, 0, None, ME, True), tr(b - 5, False, 0, 10.0, ME, False)), 0, 0.0))
        elif kind == 1:
            cuts.append(Cut(f"b{c}", MIX, LINEAR, (tr(np.abs(a) + 0.1, False, 0, float(c % 7), ME, False),
                                                    tr(np.abs(b) + 0.1, False, 0, None, E, True)), 0, 0.0))
        elif kind == 2:
            cuts.append(Cut(f"b{c}", MIX, LOG, (tr(a - 4, False, 0, 3.0, ME, False), tr(b - 6, False, 1, None, ME, True)), -1, 0.0))
        else:
            cuts.append(Cut(f"b{c}", COPY, LOG, (tr(a, False, 0, None, M, False),), 0, 0.0))
    return cuts


BATCH_SIZES = [127, 128, 129, 255, 257, 65535, 65540]


# ---- what a row reaches, read from its data -------------------------------------------------------------------------------

def branches(cut, evaluated):
    """The branches `cut` reaches, from its tracks and its float64 evaluation `evaluated` (T, F)."""
    out = set()
    nr = cut.num_rows()
    if cut.mode == COPY:
        x = cut.tracks[0].rows64()
        out |= {"copy_nan"} if np.isnan(x).any() else set()
        out |= {"copy_pos_inf"} if np.isposinf(x).any() else set()
        out |= {"copy_neg_inf"} if np.isneginf(x).any() else set()
        out |= {"copy_neg_zero"} if (np.signbit(x) & (x == 0)).any() or math.copysign(1, cut.pad_value) < 0 else set()
        return out
    law, trs, k_ref = cut.law, cut.tracks, cut.ref_k()
    ref, first = trs[k_ref], trs[0]
    out.add({-1: "trim", 0: "equal", 1: "repeat"}[cut.adjust])
    if k_ref == 0:
        out.add("ref_first")
    elif ref.num_rows == 0:
        out.add("ref_zero_rows")
    elif ref.flags == E:
        out.add("ref_muted")
    else:
        out.add("ref_later_snr" if ref.snr is not None else "ref_later_no_snr")
    with np.errstate(all="ignore"):
        e_ref = FC.law_energy(law, ref.rows64())
        if k_ref != 0 and first.snr is not None:
            e0 = FC.law_energy(law, first.rows64())
            if math.isnan(e_ref):
                out.add("first_e_ref_nan")
            elif e_ref <= 0:
                out.add("first_e_ref_le0")
            elif math.isnan(e0):
                out.add("first_e0_nan")
            elif e0 <= 0:
                out.add("first_e0_le0")
            elif e0 == math.inf:
                out.add("first_e0_inf")
            else:
                out.add("first_scaled")
                g = e_ref * 10.0 ** (-first.snr / 10) / e0
                out.add("first_gain_inf" if g == math.inf else "first_gain_finite")
        for t in trs[1:]:
            if t.flags & M and t.snr is not None and e_ref > 0:
                e = FC.law_energy(law, t.rows64())
                if e > 0:
                    g = e_ref * 10.0 ** (-t.snr / 10) / e
                    out |= {"later_gain_0"} if g == 0 else {"later_gain_inf"} if g == math.inf else set()
    further = [t for t in trs[1:] if t.flags & M]
    if not further:
        out.add("not_added")
    mr = cut.mix_rows()
    covered = np.zeros(mr, bool)
    covered[: first.num_rows] = True
    for t in further:
        covered[t.offset: t.offset + t.num_rows] = True
        if t.offset >= first.num_rows:
            out.add("past_base_end")
        if t.offset == mr - 1:
            out.add("offset_last_row")
    if not covered.all():
        out.add("gap")
    v = evaluated[:nr]
    if law == LOG and further:
        at = v == LOG_EPS
        if at.any() and not at.all():
            out.add("clamp_partial")
        near = np.abs(v - LOG_EPS) < 0.6
        if (near & ~at).any():
            out.add("near_eps")
        assert not (np.abs(v[~at] - LOG_EPS) <= 1e-9 * abs(LOG_EPS)).any(), (cut.name, "an element within 1e-9 of the clamp")
    for what, test in (("nan", np.isnan), ("pos_inf", np.isposinf), ("neg_inf", np.isneginf)):
        if test(first.x if not isinstance(first.x, Const) else np.zeros(0)).any():
            out.add(f"base_{what}")
        if any(not isinstance(t.x, Const) and test(t.x).any() for t in further):
            out.add(f"further_{what}")
        if k_ref != 0 and test(ref.rows64()).any():
            out.add(f"ref_{what}")
    return out


REQUIRED_BOTH_LAWS = {"ref_first", "ref_later_no_snr", "ref_later_snr", "ref_muted", "ref_zero_rows", "first_scaled",
                      "first_e_ref_le0", "first_e0_le0", "first_e_ref_nan", "first_e0_nan", "first_e0_inf", "first_gain_inf",
                      "later_gain_0", "later_gain_inf", "not_added", "gap", "past_base_end", "offset_last_row", "trim", "equal",
                      "repeat"} | {f"{w}_{v}" for w in ("base", "further", "ref") for v in ("nan", "pos_inf", "neg_inf")}
REQUIRED_LOG = {"clamp_partial", "near_eps"}
REQUIRED_COPY = {"copy_nan", "copy_pos_inf", "copy_neg_inf", "copy_neg_zero"}
