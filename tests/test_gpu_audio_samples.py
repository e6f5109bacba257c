"""FusedAudioSamples and the audio collation kernel (csrc/collate.cuh) on the GPU: every staged route against lhotse's
collate_audio under torch.equal; reverb and generated-RIR batches against a float64 restatement of the same draws, within the
§3.1j bound per waveform sample; the kernel at its edges through the engine against a torch restatement with a NaN-filled
output; K2SpeechRecognitionDataset against lhotse's AudioSamples; and the in-model front end (B200Fbank.extract_batch on the
batch) against FusedOnTheFlyFeatures, with a gradient reaching the audio."""
import copy
import random

import numpy as np
import pytest
import torch

import audio_samples_cases as AC
import reverb_cases as RC
from test_gpu_reverb import _cases as reverb_cases
from test_gpu_reverb import _pre_reverb, _read
from test_gpu_reverb import env  # noqa: F401  (the WAV + FLAC backend, speech cuts, RIRs and the golden FLAC cut)

pytestmark = pytest.mark.gpu


def _restated(src, offsets, lens, T):
    """torch restatement: zeros, then each row's samples (int16 widened as q / 32768)."""
    x = src.float() * (1.0 / 32768.0) if src.dtype == torch.int16 else src
    out = torch.zeros((len(lens), T), dtype=torch.float32, device=src.device)
    for b, (o, n) in enumerate(zip(offsets, lens)):
        out[b, :n] = x[o: o + n]
    return out


def _launch(src, offsets, lens, T, shift=0):
    """engine.collate_audio into a (B, T) view `shift` floats into a NaN-filled buffer with 64 NaN sentinels past it."""
    from lhotse_b200 import engine as E

    B = len(lens)
    big = torch.full((shift + B * T + 64,), float("nan"), dtype=torch.float32, device="cuda:0")
    out = big[shift: shift + B * T].view(B, T)
    E.collate_audio(src, offsets, lens, out)
    torch.cuda.synchronize()
    assert torch.isnan(big[:shift]).all() and torch.isnan(big[shift + B * T:]).all()  # nothing outside the output
    assert not torch.isnan(out).any()  # every element written
    return out


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_kernel_edges_against_torch(dtype):
    rs = np.random.RandomState(1)
    for T, src, offs, lens in AC.edge_table(rs, dtype):
        s = torch.from_numpy(src).cuda()
        want = _restated(s, offs, lens, T)
        for shift in range(4):  # every alignment of the output's start, so every row-start alignment for every T
            got = _launch(s, offs, lens, T, shift)
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (T, shift)


def test_kernel_one_row_many_rows_and_long_rows():
    rs = np.random.RandomState(2)
    q = torch.from_numpy(rs.randint(-32768, 32768, size=400_000).astype(np.int16)).cuda()
    # B = 1, T = 1
    assert torch.equal(_launch(q, [0], [1], 1), _restated(q, [0], [1], 1))
    assert torch.equal(_launch(q, [8], [0], 1), torch.zeros(1, 1, device="cuda:0"))
    # a row that takes many CTAs in x, with a head and a tail
    for T, n in ((300_001, 299_999), (262_147, 262_147), (1025, 0)):
        for shift in (0, 1, 3):
            assert torch.equal(_launch(q, [4], [n], T, shift), _restated(q, [4], [n], T)), (T, n, shift)
    # more rows than one grid covers in y (65535): the rows stride
    B = 65540
    lens = [(b * 7) % 6 for b in range(B)]
    offs = [(b * 13) % 1000 for b in range(B)]
    f = torch.from_numpy(rs.randn(2000).astype(np.float32)).cuda()
    for T in (5, 6):
        got = _launch(f, offs, lens, T, shift=1)
        assert torch.equal(got, _restated(f, offs, lens, T)), T
    # no rows, no columns: nothing launched, nothing refused
    from lhotse_b200 import engine as E

    E.collate_audio(f, [], [], torch.empty((0, 7), device="cuda:0"))
    E.collate_audio(f, [0, 0], [0, 0], torch.empty((2, 0), device="cuda:0"))


def test_kernel_refusals_raise():
    from lhotse_b200 import engine as E

    f = torch.zeros(16, device="cuda:0")
    with pytest.raises(E.B200FeatError, match="length 9 above T = 8"):
        E.collate_audio(f, [0], [9], torch.empty((1, 8), device="cuda:0"))
    with pytest.raises(E.B200FeatError, match="outside the source buffer"):
        E.collate_audio(f, [12], [8], torch.empty((1, 8), device="cuda:0"))


def _equal_to_lhotse(strategy, cuts, route, **kw):
    from lhotse import CutSet
    from lhotse.dataset.collation import collate_audio

    cuts = CutSet.from_cuts(cuts)
    audio, lens = strategy(cuts)
    assert strategy.last_batch_route == route, (route, strategy.last_batch_route, strategy.last_decline)
    ref, ref_lens = collate_audio(cuts, **kw)
    assert audio.is_cuda and audio.dtype == torch.float32
    assert torch.equal(lens, ref_lens) and lens.dtype == torch.int32
    assert audio.shape == ref.shape and torch.equal(audio.cpu().view(torch.int32), ref.view(torch.int32)), route
    return audio, lens


def test_every_staged_route_equals_collate_audio(env):  # noqa: F811
    from lhotse import CutSet
    from lhotse.dataset.cut_transforms import CutMix

    from lhotse_b200 import FusedAudioSamples

    _, speech, _, fl = env
    c0, c1, c2 = speech
    sr = 16000
    plain = [c0, c1, c2.truncate(duration=3.0 - 1 / sr), c0.truncate(offset=0.1, duration=3.0 - 5 / sr)]
    st = FusedAudioSamples()
    _equal_to_lhotse(st, plain, "pcm16")
    _equal_to_lhotse(st, plain[::-1], "pcm16")  # the ring again
    flac = [fl[0].truncate(offset=1.0, duration=4.0), fl[0].truncate(offset=0.3, duration=2.0 - 3 / sr),
            fl[0].truncate(duration=4.0 - 1 / sr)]
    _equal_to_lhotse(st, flac, "flac")
    noise = CutSet.from_cuts([c2.truncate(duration=1.0, preserve_id=False), c1])
    mixed = list(CutMix(cuts=noise, p=1.0, snr=(10, 20), seed=3)(CutSet.from_cuts(plain)))
    _equal_to_lhotse(st, mixed, "mix")
    _equal_to_lhotse(st, [c0.pad(duration=4.5), c1.append(c2), c2, c0.mix(c1, snr=5, allow_padding=True)], "mix")
    perturbed = [c0.perturb_speed(1.1).mix(c1, snr=10, allow_padding=True), c1, c2.perturb_volume(0.7)]
    _equal_to_lhotse(FusedAudioSamples(perturbed_tracks=True), perturbed, "mix")
    transform = [c0.perturb_speed(0.9), c1.perturb_speed(1.1), c2.perturb_volume(1.4), c1, fl[0].truncate(duration=3.0).perturb_speed(0.9)]
    _equal_to_lhotse(st, transform, "transform")
    _equal_to_lhotse(st, [c.resample(8000) for c in plain], "transform")
    # mono_downmix=False: (B, 1, T); audio_on_device=False: on the CPU; fault_tolerant: lhotse's padded cuts back
    a, _ = FusedAudioSamples(mono_downmix=False)(CutSet.from_cuts(plain))
    from lhotse.dataset.collation import collate_audio

    ref, _ = collate_audio(CutSet.from_cuts(plain), mono_downmix=False)
    assert a.shape == ref.shape == (4, 1, ref.shape[2]) and torch.equal(a.cpu(), ref)
    a, _ = FusedAudioSamples(audio_on_device=False)(CutSet.from_cuts(plain))
    assert a.device.type == "cpu" and torch.equal(a, collate_audio(CutSet.from_cuts(plain))[0])
    a, l, kept = FusedAudioSamples(fault_tolerant=True)(CutSet.from_cuts(plain))
    ra, rl, rkept = collate_audio(CutSet.from_cuts(plain), fault_tolerant=True)
    assert torch.equal(a.cpu(), ra) and torch.equal(l, rl)
    # the same padded cuts (their PaddingCuts' ids are random UUIDs, so everything else is compared)
    assert [(c.id, type(c).__name__, c.duration, c.num_samples) for c in kept] == [
        (c.id, type(c).__name__, c.duration, c.num_samples) for c in rkept]


def _rows_within_bound(audio, lens, cuts, truth_of):
    host = audio.cpu().numpy()
    for i, c in enumerate(cuts):
        n = int(lens[i])
        assert not host[i, n:].any(), c.id
        truth, ref32 = truth_of(c)
        if truth is None:
            assert np.array_equal(host[i, :n].view(np.int32), ref32.view(np.int32)), c.id
        else:
            RC.check(host[i, :n], truth, ref32, c.id)


def test_reverb_rows_within_the_float64_bound(env):  # noqa: F811
    from lhotse import CutSet

    from lhotse_b200 import FusedAudioSamples
    from lhotse_b200.pcm_staging import transform_request_for_cut

    _, speech, rirs, fl = env
    cases = {k: v for k, v in reverb_cases(speech, rirs, fl).items() if k != "stereo_rir_ch1"}  # the WAV backend is mono
    cuts = [cases[k] for k in sorted(cases)]
    st = FusedAudioSamples(reverb=True)
    audio, lens = st(CutSet.from_cuts(cuts))
    assert st.last_batch_route == "transform"

    def truth_of(c):
        req = transform_request_for_cut(c, reverb=True)
        if req is None or req.reverb is None:
            return None, AC.load_f32(c)
        x, q = _pre_reverb(req), _read(req.reverb.rir)
        return RC.truth64(x, q, req.reverb.normalize, c.num_samples), RC.lhotse32(x, q, req.reverb.normalize, c.num_samples)

    _rows_within_bound(audio, lens, cuts, truth_of)
    assert FusedAudioSamples()(CutSet.from_cuts(cuts)) is not None  # without reverb=True: lhotse's batch
    # a MixedCut reverberated after its mix
    c0, c1, c2 = speech
    mixed = [c0.mix(c1, snr=10, allow_padding=True).reverb_rir(rirs["rir_short"]), c2]
    st = FusedAudioSamples(reverb=True)
    audio, lens = st(CutSet.from_cuts(mixed))
    assert st.last_batch_route == "mix"
    from lhotse.utils import fastcopy

    def truth_mix(c):
        if getattr(c, "tracks", None) is None:
            return None, AC.load_f32(c)
        x = np.asarray(fastcopy(c, transforms=None).load_audio(), np.float32)[0]
        t = c.transforms[-1]
        from lhotse import MonoCut

        from lhotse_b200.pcm_staging import slice_request_for_cut

        rec = t.rir
        q = _read(slice_request_for_cut(MonoCut(id="r", start=0.0, duration=rec.duration, channel=0, recording=rec)))
        return RC.truth64(x, q, t.normalize_output, c.num_samples), RC.lhotse32(x, q, t.normalize_output, c.num_samples)

    _rows_within_bound(audio, lens, mixed, truth_mix)


def test_generated_rir_rows_within_the_float64_bound(env):  # noqa: F811
    import test_gpu_rirgen as GR
    from lhotse import CutSet

    from lhotse_b200 import FusedAudioSamples

    _, speech, _, _ = env
    c0, c1, c2 = speech
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        for route, batch in (("transform", [c0.reverb_rir(room_rng_seed=1), c1.perturb_speed(1.1).reverb_rir(room_rng_seed=2), c2]),
                             ("mix", [c0.mix(c1, snr=10, allow_padding=True).reverb_rir(room_rng_seed=3),
                                      c2.reverb_rir(room_rng_seed=4), c1])):
            torch.manual_seed(3)
            state = torch.get_rng_state()
            rirs_cuts = copy.deepcopy(batch)
            rirs = GR._rirs_for(rirs_cuts, state)
            torch.set_rng_state(state)
            st = FusedAudioSamples(generated_rir=True, perturbed_tracks=True)
            audio, lens = st(CutSet.from_cuts(copy.deepcopy(batch)))
            assert st.last_batch_route == route
            after = torch.get_rng_state()
            torch.set_rng_state(state)
            for c in copy.deepcopy(batch):
                c.load_audio()
            assert torch.equal(torch.get_rng_state(), after)  # the same draws as lhotse's

            def truth_of(c):
                truth, ref32 = GR._truth(c, rirs)
                return (None, ref32) if GR._reverb_of(c) is None else (truth, ref32)

            _rows_within_bound(audio, lens, rirs_cuts, truth_of)
    finally:
        torch.set_num_threads(threads)


def test_k2_dataset_equals_audio_samples(env, tmp_path):  # noqa: F811
    import lhotse_env
    from lhotse import CutSet
    from lhotse.dataset import DynamicBucketingSampler, K2SpeechRecognitionDataset
    from lhotse.dataset.cut_transforms import CutMix, PerturbSpeed
    from lhotse.dataset.input_strategies import AudioSamples

    from lhotse_b200 import FusedAudioSamples

    rs = np.random.RandomState(0)
    cuts = lhotse_env.make_cutset(tmp_path, np.round(rs.uniform(1.0, 6.0, size=24), 3).tolist(), seed=1)
    noise = CutSet.from_cuts(lhotse_env.make_cutset(tmp_path, [2.0, 5.0], seed=7, amp=0.05, prefix="nz"))
    got, routes = {}, set()
    for name, strategy in (("reference", AudioSamples()), ("fused", FusedAudioSamples())):
        sampler = DynamicBucketingSampler(cuts, max_duration=20.0, num_buckets=2, shuffle=True, seed=0)
        ds = K2SpeechRecognitionDataset(input_strategy=strategy, return_cuts=True,
                                        cut_transforms=[CutMix(cuts=noise, p=0.5, snr=(10, 20), preserve_id=True, seed=5),
                                                        PerturbSpeed(factors=[0.9, 1.1], p=0.5, randgen=random.Random(6))])
        out = []
        for batch_cuts in sampler:
            b = ds[batch_cuts]
            sup = b["supervisions"]
            out.append((b["inputs"].cpu(), sup["start_sample"].clone(), sup["num_samples"].clone(), sup["sequence_idx"].clone(),
                        [c.id for c in sup["cut"]]))
            if name == "fused":
                routes.add(strategy.last_batch_route)
        got[name] = out
    assert routes <= {"pcm16", "mix", "transform", "reference"} and routes & {"mix", "transform"}, routes
    assert len(got["reference"]) == len(got["fused"]) > 1
    for r, f in zip(got["reference"], got["fused"]):
        assert r[4] == f[4]
        for x, y in zip(r[:4], f[:4]):
            assert torch.equal(x, y)


def test_in_model_front_end_equals_fused_features_and_backpropagates(env):  # noqa: F811
    from lhotse import CutSet

    from lhotse_b200 import FusedAudioSamples
    from lhotse_b200.input_strategies import FusedOnTheFlyFeatures

    lb_ex, speech, _, _ = env
    c0, c1, c2 = speech
    cuts = CutSet.from_cuts([c0, c1.truncate(duration=2.0), c2, c0.truncate(offset=0.5, duration=1.3)])
    st = FusedAudioSamples()
    audio, lens = st(cuts)
    assert st.last_batch_route == "pcm16"
    fbank = lb_ex.B200Fbank(lb_ex.B200FbankConfig(device="cuda:0", dither=0.0))
    rows = fbank.extract_batch(audio, 16000, lengths=lens)
    feats, feat_lens = FusedOnTheFlyFeatures(fbank)(cuts)
    for i, r in enumerate(rows):
        assert r.shape[0] == int(feat_lens[i])
        assert torch.equal(r, feats[i, : r.shape[0]]), i
    x = audio.clone().requires_grad_()
    out = fbank.extract_batch(x, 16000, lengths=lens)
    sum(r.square().mean() for r in out).backward()
    assert x.grad is not None and x.grad.shape == x.shape and bool(x.grad.abs().sum() > 0)
    for i, n in enumerate(lens.tolist()):
        assert not x.grad[i, n:].any()  # the padding is not part of any cut
