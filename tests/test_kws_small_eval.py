"""KWSModel's speech_commands nets on the GPU (--architecture low_latency_conv / tiny_conv on the DS-CNN handle): the conv and the
logits against the fp64 oracle (kws_small_oracle) with the kernels each call launches, at the reference's geometries and at each
edge the handle accepts; batch invariance across the conv's tiles and the head's K chunks and utterance groups; class counts; the
wav input paths and the listener against the forward bit for bit; the deployable and streaming models, listen_audio.py and
evaluate_audio.py end to end."""
import ctypes as C
import shlex

import numpy as np
import pytest

import kws_small_oracle as S
from oracle import metrics_oracle as MO
from oracle import tcr_oracle as O
from tcr_harness import launched
from test_dscnn import features
from test_dscnn_eval import FRONTENDS, Ds, check_parity, clips
from test_dscnn_listener import DsListener, check_ds_push
from test_kws_eval import KwsDs
from test_kws_geometry import _counts, _forward_one
from test_kws_small import SmallNet, check_small, create

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

pytestmark = pytest.mark.gpu

CONV = {"low_latency_conv": "kws_llconv", "tiny_conv": "kws_tinyconv"}
ARCHS = pytest.mark.parametrize("arch", ["low_latency_conv", "tiny_conv"])


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def check_cuda(net, feat, rows=None):
    """check_small on the GPU (the oracle on `rows`), with the kernels the conv and the forward launch named (the launch
    profiler's counts).  Returns the layer error and the logits error."""
    def layer_output():
        got = {}
        counts = launched(net.lib, lambda: got.setdefault("a", net.layer_output(feat)))
        assert counts == {CONV[net.arch]: 1}, counts
        return got["a"]
    errs = check_small(net, feat, layer_output, rows)
    counts = launched(net.lib, lambda: net.forward(feat))
    assert counts == {CONV[net.arch]: 1, "kws_fcs": 1, "kws_fcb_head": 1}, counts
    return errs


# (arch, T, F, feature kind): the reference's geometries, then the edges: low_latency_conv at F = 8 (one output column) and at
# 6400 x 8 (K = 51,200 taps in one fmaf chain) and 400 x 128 (the head's K = 22,506); tiny_conv at 1 x 1, odd / even T and F, and
# 400 x 128 (the head's K = 102,400 in 400 chunks)
GEOMETRIES = [(a, 49, 40, "mfcc") for a in CONV] + [(a, 98, 40, "mfcc") for a in CONV] + [(a, 49, 64, "logmel") for a in CONV] + [
    ("low_latency_conv", 49, 8, "randn"), ("low_latency_conv", 6400, 8, "randn"), ("low_latency_conv", 400, 128, "randn"),
    ("tiny_conv", 1, 1, "randn"), ("tiny_conv", 5, 7, "randn"), ("tiny_conv", 98, 41, "randn"), ("tiny_conv", 400, 128, "randn")]


@pytest.mark.parametrize("arch,T,Fq,kind", GEOMETRIES, ids=[f"{a}-{t}x{f}-{k}" for a, t, f, k in GEOMETRIES])
def test_cuda_layer_and_logits_match_the_oracle(cuda, arch, T, Fq, kind):
    """n = 1, 3, 39 and 512 = max_batch.  The logits of an utterance are the same bits in any batch: permuted, and on a handle
    with another max_batch."""
    big = SmallNet(cuda, arch, T, Fq, 512, seed=1)
    small = SmallNet(cuda, arch, T, Fq, 39, seed=1)
    try:
        for n in (1, 3, 39, 512):
            feat = features(kind, n, T, Fq, seed=n)
            check_cuda(big, feat)
            if n == 39:
                ref, _ = big.forward(feat)
                perm = np.random.RandomState(n).permutation(n)
                assert np.array_equal(big.forward(np.ascontiguousarray(feat[perm]))[0], ref[perm])
                assert np.array_equal(small.forward(feat)[0], ref)
    finally:
        big.close()
        small.close()


@ARCHS
def test_cuda_batch_invariance_across_tiles_and_chunks(cuda, arch):
    """Batches that end one past a full kws_llconv tile of 128 rows (49 x 40: 33 rows an utterance), a kws_fcs group of 64 and a
    kws_fcb_head group of 16, and a batch past the device's SM count of conv tiles: every utterance equals its own forward alone."""
    net = SmallNet(cuda, arch, 49, 40, 5000, seed=7)
    try:
        feat = features("randn", 5000, 49, 40, seed=9)
        full = net.forward(feat)[0]
        for n in (17, 65, 129, 4097, 5000):
            got = net.forward(np.ascontiguousarray(feat[:n]))[0]
            assert np.array_equal(got, full[:n]), n
        alone = np.concatenate([net.forward(feat[u:u + 1])[0] for u in (0, 16, 63, 64, 128, 4096, 4999)])
        assert np.array_equal(alone, full[[0, 16, 63, 64, 128, 4096, 4999]])
    finally:
        net.close()


@ARCHS
@pytest.mark.parametrize("classes", [1, 2, 17, 32])
def test_cuda_class_counts(cuda, arch, classes):
    """n = 18: the head kernel's groups of 16 utterances, a full one and a partial one.  Logits-only and probs-only calls, and the
    evaluation counts of the logits against metrics_oracle's top-k counts."""
    n = 18
    net = SmallNet(cuda, arch, 49, 40, n, seed=classes, classes=classes)
    try:
        feat = features("mfcc", n, 49, 40, seed=classes)
        check_cuda(net, feat)
        logits, probs = net.forward(feat)
        assert logits.shape == probs.shape == (n, classes)
        assert np.array_equal(_forward_one(net, feat, True, False)[0], logits), "logits-only call"
        assert np.array_equal(_forward_one(net, feat, False, True)[1], probs), "probs-only call"
        onehot = np.eye(classes, dtype=np.float32)[np.random.RandomState(classes).randint(0, classes, n)]
        for topk in (1, 5):
            got = _counts(net, logits, onehot, topk)
            assert np.array_equal(got, MO.eval_counts(logits, onehot, topk)), topk
            assert got[-1] == n
    finally:
        net.close()


class SmallDs(Ds):
    """test_dscnn_eval.Ds on a low_latency_conv / tiny_conv handle: the front-end, kws_small_oracle's seeded variables and its fp64
    logits."""

    def __init__(self, b, arch, frontend, max_batch, seed=0, classes=12):
        self.b, self.lib, self.arch = b, b.lib, arch
        c = L.TcrConfig()
        L.check(self.lib, self.lib.tcr_config_default(C.byref(c)), "tcr_config_default")
        for k, v in frontend.items():
            setattr(c, k, v)
        c.num_classes = classes
        self.cfg = c
        T = 1 + (c.clip_samples - c.window_size_samples) // c.window_stride_samples
        F = c.num_mfccs if c.feature_kind == L.TCR_FEATURE_MFCC else c.num_mel_bins
        self.T, self.F, self.classes, self.size = T, F, classes, S.CODES[arch]
        self.info = type("Info", (), dict(frames=T, features=F))
        rc, self.h = create(self.lib, arch, T, F, max_batch, classes)
        L.check(self.lib, rc, "tcr_dscnn_create")
        L.check(self.lib, self.lib.tcr_dscnn_set_frontend(self.h, C.byref(c)), "tcr_dscnn_set_frontend")
        self.spec = S.build_spec(arch, T, F, classes)
        self.p64 = S.init_variables(self.spec, seed)
        self.params = b.upload(S.flatten(self.spec, self.p64))

    def oracle_logits(self, wav):
        c = self.cfg
        x = wav.astype(np.float64) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float64)
        kw = dict(num_mel_bins=c.num_mel_bins, sample_rate=c.sample_rate, lower_edge_hertz=c.lower_edge_hertz,
                  upper_edge_hertz=c.upper_edge_hertz)
        if c.feature_kind == L.TCR_FEATURE_MFCC:
            feat = O.mfcc(x, c.window_size_samples, c.window_stride_samples, num_mfccs=c.num_mfccs, **kw)
        else:
            feat = O.log_mel_spectrogram(x, c.window_size_samples, c.window_stride_samples, magnitude_squared=False, **kw)
        return S.forward(self.spec, self.p64, feat)


@ARCHS
@pytest.mark.parametrize("case", ["49x40", "98x40"])
def test_cuda_wav_forward_matches_features_and_oracle(cuda, arch, case):
    """fp32 and int16 clips: the forward from wav equals the forward on tcr_dscnn_mfcc_forward's features bit for bit, and the fp64
    front-end + oracle within 1e-4 (40 rows of each batch)."""
    ds = SmallDs(cuda, arch, FRONTENDS[case], 512, seed=5)
    try:
        for n, pcm in ((1, False), (3, True), (39, False), (512, True)):
            rows = np.unique(np.r_[np.arange(min(n, 32)), np.arange(max(0, n - 8), n)])
            check_parity(ds, clips(n, seed=n, pcm=pcm), rows)
    finally:
        ds.close()


def run_listener(b, arch, S_, hop, K_, pushes, reset_at=(), pcm_every=3, seed=0, case="49x40"):
    """Pushes against the forward on the cut clips (listener_cases.Offline), then the windowed conv named in a push's launches.
    case: a FRONTENDS key or a dict of tcr_config front-end fields.  The launch check needs the CUDA build's profiler."""
    from listener_cases import Offline, random_chunk
    ds = SmallDs(b, arch, FRONTENDS[case] if isinstance(case, str) else case, S_ * K_, seed=seed)
    lis = DsListener(ds, S_, hop, K_ * hop * ds.cfg.window_stride_samples)
    try:
        off = Offline(ds, S_, hop)
        rng = np.random.default_rng(seed)
        for i in range(pushes):
            for r in (x for at, x in reset_at if at == i):
                lis.reset(r)
                for s in (range(S_) if r == -1 else [r]):
                    off.reset(s)
            check_ds_push(ds, lis, off, random_chunk(rng, S_, lis.chunk, pcm=(i % pcm_every == pcm_every - 1)))
        if b.name == "cuda":
            got = launched(b.lib, lambda: lis.push(np.zeros((S_, lis.chunk), np.float32)))
            assert got[CONV[arch] + ":win"] == 1 and CONV[arch] not in got, got
    finally:
        lis.close()
        ds.close()


@ARCHS
def test_cuda_listener_matches_the_cut_clips(cuda, arch):
    """13 streams x 3 windows at hop = T - 1 (fp32 and int16 pushes, reset of every stream and of the last one), K = hop = 1, and
    98 x 40 windows (tiny_conv: an even T, no row of padding below)."""
    run_listener(cuda, arch, S_=13, hop=48, K_=3, pushes=4, reset_at=((2, -1), (3, 12)), pcm_every=2)
    run_listener(cuda, arch, S_=7, hop=1, K_=1, pushes=5, pcm_every=2)
    run_listener(cuda, arch, S_=3, hop=5, K_=2, pushes=3, case="98x40")


def test_cuda_small_listeners_interleave_with_trad_fpool3(cuda):
    """A low_latency_conv, a tiny_conv and a trad_fpool3 listener pushed in turn: each keeps its own state and matches its own
    model."""
    from listener_cases import Offline, random_chunk
    dss = [SmallDs(cuda, "low_latency_conv", FRONTENDS["49x40"], 6, seed=1), SmallDs(cuda, "tiny_conv", FRONTENDS["49x40"], 6, seed=2),
           KwsDs(cuda, "trad_fpool3", FRONTENDS["49x40"], 6, seed=3)]
    lis = [DsListener(d, 2, 3, 3 * 3 * d.cfg.window_stride_samples) for d in dss]
    try:
        offs = [Offline(d, 2, 3) for d in dss]
        rng = np.random.default_rng(3)
        for i in range(4):
            for d, l, o in zip(dss, lis, offs):
                check_ds_push(d, l, o, random_chunk(rng, 2, l.chunk, pcm=i == 2))
    finally:
        for l in lis:
            l.close()
        for d in dss:
            d.close()


def _flags(arch):
    return ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
            f"--window_size_ms 40 --window_stride_ms 20", f"KWSModel --architecture {arch}")


@ARCHS
def test_deployed_and_streaming_models_and_listen_audio(cuda, tmp_path, arch):
    """build_deployable_model: eager calls then graph replay, each equal to forward_input on the clip; build_streaming_model pushes
    equal to forward_input on the cut clips; listen_audio.py on a checkpoint under the bare names writes one .npy and .csv per
    file, the softmaxes of the forward on its windows."""
    import torch
    from listener_cases import Offline, random_chunk
    from test_listener import _write_wav
    from tcresnet_b200 import evaluate_audio, listen_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.factory import audio_nets
    flags, model = _flags(arch)
    args = evaluate_audio.parse_arguments(shlex.split(f"--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x "
                                                      f"--batch_size 1 --augmentation_method anchored_slice_or_pad {flags} {model}"))
    m = audio_nets.KWSModel(args, None)
    _, dep = m.build_deployable_model(include_preprocess=True)
    for i in range(4):
        x = clips(1, seed=10 + i)
        assert np.array_equal(dep(x), m.engine.forward_input(torch.from_numpy(x).cuda(), m.params)[1].cpu().numpy()), i
    assert dep._graph is not None
    sm = m.build_streaming_model(streams=3, hop_ms=40, chunk_ms=120)
    off = Offline(type("E", (), dict(cfg=sm.engine.cfg, info=sm.engine.info)), 3, 2)
    rng = np.random.default_rng(0)
    for i in range(4):
        x = random_chunk(rng, 3, sm.chunk_samples, pcm=i == 2)
        got = sm(x)
        cut = off.push(x).reshape(9, -1)
        ref = sm.engine.forward_input(torch.from_numpy(cut).cuda(), m.params)[1].cpu().numpy().reshape(3, 3, -1)
        assert np.array_equal(got, ref), i
    sm.listener.close()
    spec = S.build_spec(arch, 49, 40, 12)
    values = {k: v.astype(np.float32) for k, v in S.init_variables(spec, 2).items()}
    path = ckpt.save(tmp_path / "run", "KWSModel", 100, values, fmt="tf")
    wavs = []
    for name in ("a", "b"):
        wav = rng.integers(-20000, 20000, 12000).astype(np.int16)
        _write_wav(tmp_path / f"{name}.wav", wav)
        wavs.append(wav)
    out = tmp_path / "out"
    la = listen_audio.parse_arguments(shlex.split(f"--checkpoint_path {path} --hop_ms 40 --chunk_ms 120 --output_dir {out} "
                                                  f"{flags} {model} {tmp_path / 'a.wav'} {tmp_path / 'b.wav'}"))
    results = listen_audio.listen(la)
    assert len(results) == 2
    for name, probs in zip(("a", "b"), results):
        assert np.array_equal(np.load(out / f"{name}.npy"), probs)
        assert (out / f"{name}.csv").is_file()
        assert probs.shape == (-(-12000 // 640), 12) and np.allclose(probs.sum(1), 1, atol=1e-5)
    m.set_variables(values)
    off = Offline(type("E", (), dict(cfg=m.engine.cfg, info=m.engine.info)), 1, 2)
    pushes = -(-results[0].shape[0] // 3)
    stream = np.zeros((1, pushes * 1920), np.float32)
    stream[0, :12000] = wavs[0].astype(np.float32) / 32768.0
    cut = np.concatenate([off.push(stream[:, p * 1920:(p + 1) * 1920]) for p in range(pushes)], axis=1)[0][:results[0].shape[0]]
    ref = np.concatenate([sm.engine.forward_input(torch.from_numpy(np.ascontiguousarray(cut[i:i + 3])).cuda(), m.params)[1].cpu().numpy()
                          for i in range(0, cut.shape[0], 3)])
    assert np.array_equal(results[0], ref)
    sm.engine.close()
    m.engine.close()


@ARCHS
def test_evaluate_audio_counts_the_oracles_predictions(tmp_path, arch):
    """The one_fstride4 recipe's evaluation flags with --architecture swapped (--batch_size 3, --valid_type once) on a small
    on-disk split and a TF-V2 bundle of seeded weights and biases under the bare names: the confusion matrix and accuracy equal the
    fp64 oracle's arg-max counts, total_loss is CE + 1e-4 * sum(v^2) / 2 over every variable, biases included, and model_loss CE;
    --use_ema scores with the /ExponentialMovingAverage shadows."""
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper
    from tcresnet_b200.runtime import Session
    flags, model = _flags(arch)
    make_split(tmp_path, "valid", per_label=3, seed=2)
    spec = S.build_spec(arch, 49, 40, 12)
    values = {k: v.astype(np.float32) for k, v in S.init_variables(spec, 11).items()}
    shadows = {k: v.astype(np.float32) for k, v in S.init_variables(spec, 12).items()}
    bundle = dict(values, **{k + "/ExponentialMovingAverage": v for k, v in shadows.items()})
    path = ckpt.save(tmp_path / "run", "KWSModel", 1000, bundle, fmt="tf")

    def args(extra=""):
        return evaluate_audio.parse_arguments(shlex.split(
            f"--dataset_path {tmp_path} --dataset_split_name valid --checkpoint_path {path} --num_silent 6 "
            "--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 3 "
            f"--no-shuffle --valid_type once --no-save_best_keeper {extra} {flags} {model}"))

    def oracle(weights):
        session = Session()
        ds = SingleLabelAudioDataWrapper(args(), session, "valid", False)
        ds.get_input_and_output_op()
        ds.setup_iterator(session, ds.placeholders, ds.data)
        cm, ces = np.zeros((12, 12)), []
        w64 = {k: np.asarray(v, np.float64) for k, v in weights.items()}
        for _ in range(ds.num_samples // 3):
            wav, hot = ds.next_batch()
            ref = S.forward(spec, w64, O.mfcc(wav[..., 0].astype(np.float64), 640, 320, num_mfccs=40))
            top2 = np.sort(ref, axis=1)[:, -2:]
            assert (top2[:, 1] - top2[:, 0]).min() > 1e-4 * np.abs(ref).max()
            np.add.at(cm, (hot.argmax(1), ref.argmax(1)), 1)
            logp = ref - ref.max(1, keepdims=True)
            logp -= np.log(np.exp(logp).sum(1, keepdims=True))
            ces.append(-(hot * logp).sum(1).mean())
        return cm, float(np.mean(ces)), 1e-4 * S.l2_loss(w64)

    for extra, weights in (("", values), ("--use_ema", shadows)):
        results = evaluate_audio.main(args(extra))
        assert len(results) == 1
        got = results[0]
        cm, ce, l2 = oracle(weights)
        assert np.array_equal(np.asarray(got["confusion_matrix"]), cm), extra
        assert got["accuracy"] == np.trace(cm) / cm.sum()
        assert abs(got["total_loss"] - (ce + l2)) <= 1e-5 * abs(ce + l2), (got["total_loss"], ce, l2)
