"""Precomputed features on the GPU: the feature-mix kernels (csrc/featmix.cuh) against the float64 evaluation of hand-built
tables at their edges (no lhotse needed), the public FusedPrecomputedFeatures against lhotse's collate_features under the
§3.1m contract, and K2SpeechRecognitionDataset with CutMix and SpecAugment on top of it."""
import math
import random

import numpy as np
import pytest
import torch

import featmix_cases as FC
import refshim

pytestmark = pytest.mark.gpu
needs_ref = pytest.mark.skipif(not refshim.reference_available(), reason="lhotse (oracle/_ref/lhotse_ref.zip) not present")

SENTINEL = np.float32(-7.75e30)


def _table(rs, F, specs, law=FC.LOG):
    """specs: one list per cut of (rows, offset, snr, flags, const, dup) -> (src, tracks, cuts, T)."""
    from lhotse_b200.engine import FEATMIX_CUT_DTYPE, FEATMIX_TRACK_DTYPE

    src, tracks, cuts = [], [], []
    elem = 0
    for c, spec in enumerate(specs):
        first = len(tracks)
        mix_rows = 0
        for k, (rows, off, snr, flags, const, dup) in enumerate(spec):
            stored = 0 if const is not None else rows - (1 if dup else 0)
            if stored:
                if law == FC.LOG:
                    x = (rs.randn(stored, F) * 2 - 5).astype(np.float32)
                elif snr == "neg":
                    x = -np.abs(rs.randn(stored, F)).astype(np.float32)
                elif snr == "zero":
                    x = np.zeros((stored, F), np.float32)
                else:
                    x = rs.randn(stored, F).astype(np.float32)
                pad = (-elem) % 4
                src.append(np.zeros(pad, np.float32))
                elem += pad
                src.append(x.ravel())
            factor = 10.0 ** (-snr / 10) if isinstance(snr, (int, float)) else math.nan
            tracks.append((FEATMIX_TRACK_DTYPE.itemsize, c, flags, stored, rows, off, 0.0 if const is None else const, 0, elem,
                           factor))
            elem += stored * F
            if flags & FC.MIXED:
                mix_rows = max(mix_rows, off + rows)
        nt = len(tracks) - first
        ref = next(k for k, s in enumerate(spec) if s[3] & FC.ENERGY)
        cuts.append((FEATMIX_CUT_DTYPE.itemsize, FC.MIX if nt > 1 or spec[0][2] is not None else FC.COPY, law, 0, mix_rows, first,
                     nt, ref, np.float32(-9.5), 0))
    cuts = np.array(cuts, dtype=FEATMIX_CUT_DTYPE)
    for c in range(len(cuts)):  # num_rows: the mix, trimmed or repeated by one for a few cuts
        cuts["num_rows"][c] = max(1, cuts["mix_rows"][c] + (c % 3) - 1) if cuts["mode"][c] == FC.MIX else cuts["mix_rows"][c] + c % 2
    T = int(cuts["num_rows"].max()) + 2
    return np.concatenate(src) if src else np.zeros(0, np.float32), np.array(tracks, dtype=FEATMIX_TRACK_DTYPE), cuts, T


def _run(src, tracks, cuts, F, T, pad=-23.025850929940457):
    from lhotse_b200 import engine as E

    dev = torch.device("cuda", 0)
    buf = torch.full((len(cuts) * T * F + 64,), float(SENTINEL), dtype=torch.float32, device=dev)
    out = buf[32: 32 + len(cuts) * T * F].view(len(cuts), T, F)
    s = torch.from_numpy(src).to(dev) if src.size else None
    E.feature_mix(s, tracks, cuts, out, pad)
    torch.cuda.synchronize()
    host = buf.cpu().numpy()
    assert (host[:32] == SENTINEL).all() and (host[32 + out.numel():] == SENTINEL).all(), "write outside the output"
    return out.cpu().numpy()


def _check(src, tracks, cuts, F, T, what):
    pad = -23.025850929940457
    got = _run(src, tracks, cuts, F, T, pad)
    again = _run(src, tracks, cuts, F, T, pad)
    assert np.array_equal(got.view(np.int32), again.view(np.int32)), f"{what}: not deterministic"
    truth = FC.evaluate(src, tracks, cuts, F, T, pad)
    err = np.abs(got.astype(np.float64) - truth)
    assert (err <= FC.ulp32(truth)).all(), (what, float(err.max()))


M, ME = FC.MIXED, FC.MIXED | FC.ENERGY


@pytest.mark.parametrize("F", [1, 80, 2500])
def test_kernels_at_chunk_and_tile_edges(F):
    rs = np.random.RandomState(F)
    per = 2048 // F if F < 2048 else 1  # rows of one energy chunk / output tile (FM_CHUNK = FM_TILE = 2048 elements)
    specs = []
    for rows in sorted({max(1, per - 1), per, per + 1, 8 * per - 1, 8 * per, 8 * per + 1, 1}):
        specs.append([(rows, 0, None, ME, None, False), (max(1, rows // 2), rows // 3, 10.0, ME, None, False)])
        specs.append([(rows, 0, 5.0, ME, None, rows > 1), (rows + 1, 0, None, ME, None, False), (3, rows, -3.0, ME, None, False)])
        specs.append([(rows, 0, None, ME, None, False), (2, 0, None, M, np.float32(-23.025851), False)])
    for law in (FC.LOG, FC.LINEAR):
        src, tracks, cuts, T = _table(rs, F, specs, law)
        _check(src, tracks, cuts, F, T, f"F={F} law={law}")


def test_zero_and_negative_energies():
    rs = np.random.RandomState(1)
    F = 80
    specs = [
        [(40, 0, None, ME, None, False), (30, 5, "zero", ME, None, False)],
        [(40, 0, "neg", ME, None, False), (30, 5, 10.0, ME, None, False)],
        [(40, 0, 3.0, ME, None, False), (30, 5, None, ME, None, False), (20, 0, "neg", ME, None, False)],
        [(0, 0, None, ME, np.float32(0.0), False), (30, 5, 10.0, ME, None, False)],  # a zero constant reference
    ]
    for law in (FC.LINEAR, FC.LOG):
        src, tracks, cuts, T = _table(rs, F, specs, law)
        _check(src, tracks, cuts, F, T, f"law={law}")


def test_thirty_tracks_and_more_cuts_than_one_gains_block():
    rs = np.random.RandomState(2)
    F = 80
    thirty = [(50, 0, None, ME, None, False)] + [(int(rs.randint(1, 40)), int(rs.randint(0, 60)), float(rs.uniform(-5, 20)),
                                                  ME, None, bool(k % 5 == 0)) for k in range(28)] + [(10, 55, None, M, np.float32(-23.025851), False)]
    specs = [thirty] + [[(int(rs.randint(1, 60)), 0, None, ME, None, False), (int(rs.randint(1, 30)), int(rs.randint(0, 20)),
                                                                               float(rs.uniform(0, 20)), ME, None, False)]
                        for _ in range(200)]
    for law in (FC.LOG, FC.LINEAR):
        src, tracks, cuts, T = _table(rs, F, specs, law)
        assert len(cuts) > 128
        _check(src, tracks, cuts, F, T, f"law={law}")


@pytest.fixture(scope="module")
def lhotse():
    if not refshim.reference_available():
        pytest.skip("lhotse (oracle/_ref/lhotse_ref.zip) not present")
    import lhotse_env

    lhotse_env.setup_lhotse()
    import lhotse

    return lhotse


@needs_ref
def test_strategy_against_collate_features(lhotse, tmp_path):
    import lhotse_b200 as lb
    from test_precomputed import batches

    strategy = lb.FusedPrecomputedFeatures(num_workers=2)
    for name, cuts in batches(tmp_path).items():
        feats, lens = strategy(cuts)
        assert strategy.last_batch_route == "archive", (name, strategy.last_decline)
        assert feats.is_cuda and feats.dtype == torch.float32 and lens.dtype == torch.int32
        again, _ = strategy(cuts)
        assert torch.equal(feats, again), name
        l32, ref_lens, truth = FC.lhotse_pair(cuts)
        assert torch.equal(lens, ref_lens)
        got = feats.cpu()
        if not (lb.precomputed_plan(cuts).cuts["mode"] == FC.MIX).any():  # no cut performs a real mix
            assert torch.equal(got, l32), name
        else:
            FC.check_gate(got.numpy(), l32.numpy(), truth.numpy(), name)


@needs_ref
def test_k2_dataset_with_cutmix_and_specaugment(lhotse, tmp_path):
    from lhotse import CutSet
    from lhotse.dataset import CutMix, DynamicBucketingSampler, K2SpeechRecognitionDataset, PrecomputedFeatures, SpecAugment

    import lhotse_b200 as lb

    cuts = FC.make_cuts(tmp_path / "a", list(np.random.RandomState(0).randint(300, 900, size=24)), seed=1)
    noise = FC.make_cuts(tmp_path / "a", [200, 1100, 450], seed=2, prefix="n", supervisions=False)
    ours_strategy = lb.FusedPrecomputedFeatures(num_workers=2)
    ours = K2SpeechRecognitionDataset(input_strategy=ours_strategy, cut_transforms=[CutMix(noise, p=0.5, snr=(10, 20), seed=7)],
                                      input_transforms=[lb.B200SpecAugment()], return_cuts=True)
    ref = K2SpeechRecognitionDataset(input_strategy=PrecomputedFeatures(), cut_transforms=[CutMix(noise, p=0.5, snr=(10, 20), seed=7)],
                                     input_transforms=[SpecAugment()])
    plain = K2SpeechRecognitionDataset(input_strategy=lb.FusedPrecomputedFeatures(),
                                       cut_transforms=[CutMix(noise, p=0.5, snr=(10, 20), seed=7)], return_cuts=True)
    sampler = DynamicBucketingSampler(cuts, max_duration=40.0, num_buckets=2, shuffle=True, seed=0)
    n = 0
    for batch in sampler:
        def seed():
            random.seed(n), np.random.seed(n), torch.manual_seed(n)

        seed()
        g = ours[batch]
        assert ours_strategy.last_batch_route == "archive", ours_strategy.last_decline
        seed()
        r = ref[batch]
        seed()
        p = plain[batch]
        # before SpecAugment: the §3.1m gate against lhotse's own collation of the same mixed cuts
        l32, _, truth = FC.lhotse_pair(CutSet.from_cuts(p["supervisions"]["cut"]))
        FC.check_gate(p["inputs"].cpu().numpy(), l32.numpy(), truth.numpy(), f"batch {n}")
        # after it: the same draws, so the same masks and warps; values within float32 noise of lhotse's
        gi, ri = g["inputs"].cpu(), r["inputs"]
        assert gi.shape == ri.shape
        torch.testing.assert_close(gi, ri, rtol=1e-5, atol=2e-4)
        for k in ("sequence_idx", "start_frame", "num_frames"):
            assert torch.equal(g["supervisions"][k], r["supervisions"][k])
        n += 1
    assert n >= 2
