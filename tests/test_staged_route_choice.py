"""`pcm_staging.staged_route`, the one route choice of `FusedOnTheFlyFeatures` and `compute_and_store_features_fused`, on real
lhotse cuts: the route each kind of batch takes, the requests it hands over (those of the per-route request functions), and
its agreement with the store's earlier pcm16 -> flac -> mix -> transform chain, written out below as the specification."""
import itertools
import os

import pytest

import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLDEN = [os.path.join(ROOT, "tests", "golden", f"2412-153948-000{i}.flac") for i in (0, 1)]


@pytest.fixture(scope="module")
def batches(tmp_path_factory):
    """name -> (cuts, the route with the default arguments, the route with perturbed_tracks=True and reverb=True)."""
    if not refshim.reference_available():
        pytest.skip("reference tree not present")
    import lhotse_env

    lhotse_env.setup_lhotse()
    import mix_cases
    import perturbed_mix_cases
    import reverb_cases
    import transform_cases
    from lhotse import Recording
    from lhotse.audio import AudioSource

    root = tmp_path_factory.mktemp("routes")
    speech, noise, s48 = perturbed_mix_cases.sources(root)
    flac = perturbed_mix_cases.flac_cuts(GOLDEN)
    mixed = mix_cases.mixed_cases(root, speech, noise)
    tsrc = transform_cases.sources(root)
    reverb_cases.write_wav(root / "rir.wav", reverb_cases.decaying_rir(4800, seed=1))
    rir = Recording(id="rir", sources=[AudioSource(type="file", channels=[0], source=str(root / "rir.wav"))],
                    sampling_rate=16000, num_samples=4800, duration=0.3)
    with transform_cases.torch_resampler():
        perturbed_mix = perturbed_mix_cases.cases(root, speech, noise, s48)["volume_track"]
    mix = next(iter(mixed.values()))
    return {
        "all_wav": ([speech[0], speech[1], noise[2]], "pcm16", "pcm16"),
        "all_flac": (flac, "flac", "flac"),
        "wav_next_to_flac": ([speech[0], flac[0]], None, None),
        "mixedcut": ([mix, speech[2]], "mix", "mix"),
        "mixedcuts_flac_beside": ([mix, flac[1]], "mix", "mix"),
        "speed_perturbed": ([speech[0].perturb_speed(1.1), speech[1]], "transform", "transform"),
        "speed_perturbed_flac": ([flac[0].perturb_speed(0.9), flac[1]], "transform", "transform"),
        "perturbed_track": ([perturbed_mix, speech[0]], None, "mix"),
        "reverberated": ([speech[0].reverb_rir(rir), speech[1]], None, "transform"),
        "two_rates": ([speech[0], tsrc[8000]], None, None),
        "two_rates_perturbed": ([speech[0].perturb_speed(1.1), tsrc[8000]], None, None),
    }


def _routes(cuts, perturbed_tracks=False, reverb=False):
    from lhotse_b200.pcm_staging import staged_route

    import transform_cases

    with transform_cases.torch_resampler():
        return staged_route(cuts, perturbed_tracks=perturbed_tracks, reverb=reverb)


def test_route_of_each_batch_kind(batches):
    for name, (cuts, plain, both) in batches.items():
        got = _routes(cuts)
        assert (got and got[0]) == plain, name
        got = _routes(cuts, perturbed_tracks=True, reverb=True)
        assert (got and got[0]) == both, name
    cuts = batches["perturbed_track"][0]
    assert _routes(cuts, perturbed_tracks=True)[0] == "mix" and _routes(cuts, reverb=True) is None
    cuts = batches["reverberated"][0]
    assert _routes(cuts, reverb=True)[0] == "transform" and _routes(cuts, perturbed_tracks=True) is None


def test_requests_are_those_of_the_route_functions(batches):
    from lhotse_b200.pcm_staging import (flac_request_for_cut, mix_requests_for_batch, pcm16_request_for_cut,
                                         transform_requests_for_batch)

    import transform_cases

    for name, (cuts, _, _) in batches.items():
        for pt, rv in itertools.product((False, True), repeat=2):
            got = _routes(cuts, perturbed_tracks=pt, reverb=rv)
            if got is None:
                continue
            with transform_cases.torch_resampler():
                want = {"pcm16": lambda: [pcm16_request_for_cut(c) for c in cuts],
                        "flac": lambda: [flac_request_for_cut(c) for c in cuts],
                        "mix": lambda: mix_requests_for_batch(cuts, perturbed_tracks=pt, reverb=rv),
                        "transform": lambda: transform_requests_for_batch(cuts, reverb=rv)}[got[0]]()
            assert want is not None and all(r is not None for r in want), (name, pt, rv)
            assert repr(got[1]) == repr(want), (name, pt, rv)  # repr: the NaN SNR factors of a mix compare unequal


def _store_chain(cuts, perturbed_tracks, reverb):
    """The route choice `compute_and_store_features_fused` made for a batch of one sampling rate before `staged_route`:
    every cut a WAV slice, else every cut a FLAC slice, else the mix requests, else the transform requests."""
    from lhotse_b200.pcm_staging import (flac_request_for_cut, mix_requests_for_batch, pcm16_request_for_cut,
                                         transform_requests_for_batch)

    kind, reqs = "pcm16", [pcm16_request_for_cut(c) for c in cuts]
    if not all(r is not None for r in reqs):
        kind, reqs = "flac", [flac_request_for_cut(c) for c in cuts]
    if not all(r is not None for r in reqs):
        kind, reqs = "mix", mix_requests_for_batch(cuts, perturbed_tracks=perturbed_tracks, reverb=reverb) or [None]
    if not all(r is not None for r in reqs):
        kind, reqs = "transform", transform_requests_for_batch(cuts, reverb=reverb) or [None]
    return (kind, reqs) if all(r is not None for r in reqs) else None


def test_agrees_with_the_store_chain(batches):
    import transform_cases

    for name, (cuts, _, _) in batches.items():
        if len({c.sampling_rate for c in cuts}) != 1:
            continue  # the store asserts one sampling rate per batch
        for pt, rv in itertools.product((False, True), repeat=2):
            with transform_cases.torch_resampler():
                want = _store_chain(cuts, pt, rv)
            assert repr(_routes(cuts, perturbed_tracks=pt, reverb=rv)) == repr(want), (name, pt, rv)
