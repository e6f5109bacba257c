"""FusedAudioSamples and the audio collation kernel without a GPU: the equivalence the design rests on (lhotse's collate_audio
is each cut's load_audio() and then zeros, with int32 cut.num_samples lengths), the NumPy restatement of csrc/collate.cuh's
row plan against it, the header's index math on the host under AddressSanitizer, the ABI's table checks (before anything
touches the device), the constructor against AudioSamples', the batches that go to lhotse, and the kernel's code generation."""
import inspect
import os
import subprocess

import numpy as np
import pytest
import torch

import audio_samples_cases as AC
import refshim

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lhotse_root(tmp_path_factory):
    if not refshim.reference_available():
        pytest.skip("no reference tree / oracle/_ref archive")
    import lhotse_env

    AC.setup_reference()
    root = tmp_path_factory.mktemp("audio_samples")
    noise = list(lhotse_env.make_cutset(root, [0.6, 1.7], seed=5, amp=0.05, prefix="n"))
    return root, noise


@pytest.fixture(scope="module")
def batches(lhotse_root):
    root, noise = lhotse_root
    return AC.lhotse_batches(root, noise)


@pytest.mark.reference
@pytest.mark.parametrize("name", ["plain", "one_short", "speed", "volume", "resample", "padding_concat", "cutmix"])
def test_collate_audio_is_load_audio_then_zeros(batches, name):
    from lhotse.dataset.collation import collate_audio

    cuts = batches[name]
    audio, lens = collate_audio(cuts)
    rows = [AC.load_f32(c) for c in cuts]
    assert audio.dtype == torch.float32 and audio.shape == (len(cuts), max(len(r) for r in rows))
    assert lens.dtype == torch.int32 and lens.tolist() == [c.num_samples for c in cuts]
    for i, r in enumerate(rows):
        assert len(r) == cuts[i].num_samples, (name, i)
        assert np.array_equal(audio[i, : len(r)].numpy().view(np.int32), r.view(np.int32)), (name, i)
        assert not audio[i, len(r):].any(), (name, i)
    if name == "cutmix":
        assert any(getattr(c, "tracks", None) is not None for c in cuts)


@pytest.mark.reference
@pytest.mark.parametrize("name", ["plain", "speed", "cutmix"])
def test_restated_kernel_equals_collate_audio(batches, name):
    from lhotse.dataset.collation import collate_audio

    cuts = batches[name]
    audio, _ = collate_audio(cuts)
    buf, offs, lens = AC.pack([AC.load_f32(c) for c in cuts], np.float32)
    for base in range(4):
        got = AC.restate(buf, offs, lens, audio.shape[1], base)
        assert np.array_equal(got.view(np.int32), audio.numpy().view(np.int32)), (name, base)


@pytest.mark.reference
def test_restated_kernel_widens_int16_as_the_float_route(batches):
    """The plain batch staged as int16 (the pcm16 route's buffer) and widened by the restatement: collate_audio's bits."""
    from lhotse.dataset.collation import collate_audio

    from lhotse_b200.pcm_staging import PcmStagingRing, staged_route

    cuts = batches["plain"]
    route, reqs = staged_route(cuts)
    assert route == "pcm16"
    staged, lens, offs, _ = PcmStagingRing(pin_memory=False).stage(reqs)
    audio, _ = collate_audio(cuts)
    got = AC.restate(staged.numpy(), offs, lens, audio.shape[1])
    assert np.array_equal(got.view(np.int32), audio.numpy().view(np.int32))


@pytest.mark.parametrize("dtype", [np.int16, np.float32])
def test_host_harness_runs_the_header_plan(tmp_path, dtype):
    exe = AC.build_harness(tmp_path)
    if exe is None:
        pytest.skip("no C++ compiler")
    rs = np.random.RandomState(7)
    for T, src, offs, lens in AC.edge_table(rs, dtype):
        for base in range(4):
            got = AC.run_harness(exe, tmp_path, src, offs, lens, T, base)
            want = AC.restate(src, offs, lens, T, base)
            assert np.array_equal(got.view(np.int32), want.view(np.int32)), (T, base)
            assert not np.isnan(got).any()


@pytest.mark.parametrize("b,T", [(0, 1), (1, 1), (3, 1), (70000, 40001), (65536, 32768), (1, (1 << 31) + 3),
                                 (2, (1 << 31) - 1), (3, (1 << 32) + 1), ((1 << 31) - 1, 7)])
def test_host_harness_plan_past_2_31(tmp_path, b, T):
    """Row plans whose row start b * T passes 2^31 (or whose T does), checked in 64-bit without allocating the rows."""
    exe = AC.build_harness(tmp_path)
    if exe is None:
        pytest.skip("no C++ compiler")
    for base in range(4):
        res = subprocess.run([exe, "--plan", str(b), str(T), str(base)], capture_output=True, text=True)
        assert res.returncode == 0, (b, T, base, res.stdout, res.stderr)
        head = int(res.stdout.split()[1])
        assert head == min((4 - (base + b * T) % 4) % 4, T)
        vectors = int(res.stdout.split()[3])
        assert vectors == (T - head) // 4


def _call(lib, dt, src_elems, offsets, lens, T, work_bytes=1 << 20):
    """b200feat_collate_audio with stand-in device pointers: only a refused table may be passed (nothing is launched)."""
    off = np.asarray(offsets, np.int64)
    ln = np.asarray(lens, np.int64)
    return lib.b200feat_collate_audio(None, 1 << 20, dt, src_elems, off.ctypes.data, ln.ctypes.data, len(off), T, 1 << 21,
                                      1 << 22, work_bytes, None)


@pytest.mark.parametrize("case,args,message", [
    ("len_above_T", (0, 100, [0, 8], [5, 11], 10), "cut 1: length 11 above T = 10"),
    ("past_source", (1, 100, [0, 92], [4, 9], 10), "cut 1: samples [92, 101) outside the source buffer of 100 elements"),
    ("negative_offset", (0, 100, [0, -4], [4, 4], 10), "cut 1: negative offset -4"),
    ("negative_length", (1, 100, [0, 4, 8], [4, 4, -1], 10), "cut 2: negative length -1"),
    ("unknown_dtype", (2, 100, [0], [4], 10), "unknown dtype 2"),
    ("negative_T", (0, 100, [0], [0], -1), "negative B, T or source size"),
    ("work_too_small", (0, 100, [0], [4], 10, 8), "work buffer too small"),
])
def test_abi_refuses_bad_tables_before_the_device(case, args, message):
    from lhotse_b200.engine import load_library

    lib = load_library()
    rc = _call(lib, *args)
    assert rc == -1, case
    assert lib.b200feat_global_error().decode() == "collate_audio: " + message, case


def test_abi_misaligned_buffers_refused():
    from lhotse_b200.engine import load_library

    lib = load_library()
    off, ln = np.zeros(1, np.int64), np.full(1, 4, np.int64)
    rc = lib.b200feat_collate_audio(None, (1 << 20) + 4, 0, 100, off.ctypes.data, ln.ctypes.data, 1, 8, 1 << 21, 1 << 22, 64, None)
    assert rc == -1 and "aligned" in lib.b200feat_global_error().decode()
    rc = lib.b200feat_collate_audio(None, 1 << 20, 1, 100, off.ctypes.data, ln.ctypes.data, 1, 8, (1 << 21) + 2, 1 << 22, 64, None)
    assert rc == -1 and "output not 4-byte aligned" in lib.b200feat_global_error().decode()
    assert lib.b200feat_collate_audio_work_bytes(5) == 80 and lib.b200feat_collate_audio_work_bytes(-1) == 0


def test_kernel_builds_without_spills():
    """Both instantiations (int16 and float32 sources) in the library build's ptxas report: no stack, no spills."""
    from lhotse_b200 import build

    log = os.path.join(build.CSRC, "ptxas.log")
    if not os.path.exists(log):
        pytest.skip("the library was not built here (no ptxas report)")
    text = open(log).read()
    found = 0
    for block in text.split("Compiling entry function")[1:]:
        name = block.split("'")[1]
        if "collate_audio_kernel" not in name:
            continue
        found += 1
        assert "0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads" in block, name
    assert found == 2


@pytest.mark.reference
def test_signature_accepts_every_audio_samples_parameter(lhotse_root):
    from lhotse.dataset.input_strategies import AudioSamples

    from lhotse_b200 import FusedAudioSamples

    ours = inspect.signature(FusedAudioSamples.__init__).parameters
    for name, p in inspect.signature(AudioSamples.__init__).parameters.items():
        assert name in ours, name
        assert ours[name].default == p.default, name
    assert list(ours)[: len(inspect.signature(AudioSamples.__init__).parameters)] == list(
        inspect.signature(AudioSamples.__init__).parameters)  # same positions
    for name, default in (("audio_on_device", True), ("perturbed_tracks", False), ("reverb", False), ("generated_rir", False)):
        assert ours[name].default is default
    call = inspect.signature(FusedAudioSamples.__call__).parameters
    assert list(call) == list(inspect.signature(AudioSamples.__call__).parameters)


@pytest.fixture
def recorder(monkeypatch, lhotse_root):
    """lhotse's collate_audio, recording each call's arguments."""
    import lhotse.dataset.collation as col

    calls = []
    real = col.collate_audio

    def spy(cuts, **kw):
        calls.append(kw)
        return real(cuts, **kw)

    monkeypatch.setattr(col, "collate_audio", spy)
    return calls


def _declined(strategy, calls, cuts, reason, **kw):
    out = strategy(cuts, **kw)
    assert strategy.last_batch_route == "reference" and reason in strategy.last_decline, strategy.last_decline
    assert len(calls) == 1
    assert calls[0]["fault_tolerant"] == strategy.fault_tolerant and calls[0]["mono_downmix"] == strategy.mono_downmix
    assert calls[0]["recording_field"] == kw.get("recording_field")
    return out


@pytest.mark.reference
def test_declined_batches_reach_lhotse(lhotse_root, recorder, tmp_path):
    import lhotse_env
    from lhotse import CutSet, MultiCut, Recording
    from lhotse.audio import AudioSource
    from lhotse.utils import fastcopy

    from lhotse_b200 import FusedAudioSamples
    from lhotse_b200.pcm_staging import staged_route

    root, _ = lhotse_root
    cuts = list(lhotse_env.make_cutset(tmp_path, [0.5, 0.3], seed=2, prefix="d"))
    # recording_field: the custom recording is the cut's own
    custom = [c.with_custom("other", c.recording) for c in cuts]
    _declined(FusedAudioSamples(audio_on_device=False), recorder, CutSet.from_cuts(custom), "recording_field",
              recording_field="other")
    recorder.clear()
    # use_batch_loader: the batch goes through the AIStore loader (a stand-in here) and then collate_audio
    st = FusedAudioSamples(audio_on_device=False)
    st.use_batch_loader, st.ais_batch_loader = True, lambda cs: cs
    _declined(st, recorder, CutSet.from_cuts(cuts), "use_batch_loader")
    recorder.clear()
    # a MultiCut over a two-channel recording (here its two channels are the same mono file)
    path = cuts[0].recording.sources[0].source
    rec = Recording(id="mc", sources=[AudioSource(type="file", channels=[0], source=path),
                                      AudioSource(type="file", channels=[1], source=path)],
                    sampling_rate=16000, num_samples=cuts[0].num_samples, duration=cuts[0].duration)
    mc = MultiCut(id="mc", start=0.0, duration=cuts[0].duration, channel=[0, 1], recording=rec)
    st = FusedAudioSamples(audio_on_device=False, mono_downmix=True)
    assert st(CutSet.from_cuts([mc, cuts[1]])) is not None
    assert st.last_batch_route == "reference" and "MultiCut" in st.last_decline
    recorder.clear()
    # two sampling rates
    _declined(FusedAudioSamples(audio_on_device=False), recorder, CutSet.from_cuts([cuts[0], cuts[1].resample(8000)]),
              "sampling rate")
    recorder.clear()
    # a cut no staged route takes: a WAV file under another extension (the staged readers choose by extension)
    import shutil

    other = tmp_path / "d0.pcm"
    shutil.copy(cuts[0].recording.sources[0].source, other)
    odd = [fastcopy(cuts[0], recording=fastcopy(cuts[0].recording, sources=[AudioSource(type="file", channels=[0],
                                                                                       source=str(other))])), cuts[1]]
    assert staged_route(odd) is None
    _declined(FusedAudioSamples(audio_on_device=False), recorder, CutSet.from_cuts(odd), "no staged route")
    recorder.clear()


@pytest.mark.reference
def test_staged_failure_declines_only_when_fault_tolerant(lhotse_root, recorder, tmp_path, monkeypatch):
    """A staged read that fails: under fault_tolerant the batch goes to lhotse (which skips what it cannot read), without it
    the error is raised."""
    import lhotse_env
    from lhotse import CutSet

    from lhotse_b200 import FusedAudioSamples
    from lhotse_b200.pcm_staging import PcmStagingRing

    cuts = CutSet.from_cuts(lhotse_env.make_cutset(tmp_path, [0.5, 0.3], seed=2, prefix="f"))

    def failing(self, reqs, executor=None):
        raise OSError("short read")

    monkeypatch.setattr(PcmStagingRing, "stage", failing)
    st = FusedAudioSamples(audio_on_device=False, fault_tolerant=True)
    out = _declined(st, recorder, cuts, "failed")
    assert len(out) == 3 and [c.id for c in out[2]] == [c.id for c in cuts]
    with pytest.raises(OSError):
        FusedAudioSamples(audio_on_device=False)(cuts)


@pytest.mark.reference
def test_reference_route_moves_audio_only_when_asked(lhotse_root, recorder, tmp_path):
    """audio_on_device=False keeps collate_audio's CPU tensors as they are; mono_downmix=False its (B, 1, T) layout."""
    import lhotse_env
    from lhotse import CutSet
    from lhotse.dataset.collation import collate_audio

    from lhotse_b200 import FusedAudioSamples

    cuts = CutSet.from_cuts(lhotse_env.make_cutset(tmp_path, [0.5, 0.3], seed=2, prefix="e"))
    st = FusedAudioSamples(audio_on_device=False, mono_downmix=False)
    custom = CutSet.from_cuts([c.with_custom("other", c.recording) for c in cuts])
    a, l = _declined(st, recorder, custom, "recording_field", recording_field="other")
    ra, rl = collate_audio(custom, recording_field="other", mono_downmix=False)
    assert a.device.type == "cpu" and a.shape == ra.shape == (2, 1, 8000) and torch.equal(a, ra) and torch.equal(l, rl)
