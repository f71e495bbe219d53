"""The KWS baselines on the GPU (KWSModel --architecture trad_fpool3 / one_fstride4 on the DS-CNN handle): each conv layer and the
logits against the fp64 oracle (kws_oracle) with the kernels each layer launches, the wav input paths and the listener against
the forward on features / cut clips bit for bit, the deployable and streaming models, listen_audio.py and evaluate_audio.py end
to end."""
import ctypes as C
import shlex

import numpy as np
import pytest

from oracle import kws_oracle as K
from oracle import tcr_oracle as O
from tcr_harness import launched, rel_err
from test_dscnn import features
from test_dscnn_eval import FRONTENDS, Ds, check_parity, clips
from test_dscnn_listener import DsListener, check_ds_push
from test_kws import KwsNet, check_net, create

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

pytestmark = pytest.mark.gpu

# launch names of each conv layer
KERNELS = {"trad_fpool3": [["kws_conv1_tc"], ["kws_bsplit", "kws_conv2_tc"]], "one_fstride4": [["kws_conv"]]}
# the windowed first layer of a listener push
WIN_KERNEL = {"trad_fpool3": "kws_conv1_tc", "one_fstride4": "kws_conv"}


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def check_layers(net, feat):
    """test_kws.check_net on the GPU, with the kernels each conv layer launches (the launch profiler's counts)."""
    seen = {}

    def layer_output(k):
        got = {}
        counts = launched(net.lib, lambda: got.setdefault("a", net.layer_output(feat, k)))
        new = counts - seen["prev"] if "prev" in seen else counts
        assert sorted(new) == KERNELS[net.arch][k - 1] and all(v == 1 for v in new.values()), (k, counts)
        seen["prev"] = counts
        return got["a"]
    return check_net(net, feat, layer_output)


@pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])
@pytest.mark.parametrize("T,Fq,kind", [(49, 40, "mfcc"), (98, 40, "mfcc"), (49, 64, "logmel"), (29, 19, "randn")],
                         ids=["49x40", "98x40", "49x64-logmel", "29x19"])
def test_cuda_layers_and_logits_match_the_oracle(cuda, arch, T, Fq, kind):
    """n = 1, 3, 39 (not a multiple of 8) and 512 = max_batch; 29 x 19 is trad_fpool3's smallest accepted geometry.  The logits of
    an utterance are the same bits in any batch: permuted, and on a handle with another max_batch."""
    big = KwsNet(cuda, arch, T, Fq, 512, seed=1)
    small = KwsNet(cuda, arch, T, Fq, 39, seed=1)
    try:
        for n in (1, 3, 39, 512):
            feat = features(kind, n, T, Fq, seed=n)
            check_layers(big, feat)
            if n == 39:
                ref, _ = big.forward(feat)
                perm = np.random.RandomState(n).permutation(n)
                assert np.array_equal(big.forward(np.ascontiguousarray(feat[perm]))[0], ref[perm])
                assert np.array_equal(small.forward(feat)[0], ref)
    finally:
        big.close()
        small.close()


class KwsDs(Ds):
    """test_dscnn_eval.Ds on a KWS handle: the front-end, kws_oracle's seeded variables and its fp64 logits."""

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
        self.T, self.F, self.classes, self.size = T, F, classes, K.CODES[arch]
        self.info = type("Info", (), dict(frames=T, features=F))
        rc, self.h = create(self.lib, arch, T, F, max_batch, classes)
        L.check(self.lib, rc, "tcr_dscnn_create")
        L.check(self.lib, self.lib.tcr_dscnn_set_frontend(self.h, C.byref(c)), "tcr_dscnn_set_frontend")
        self.spec = K.build_spec(arch, T, F, classes)
        self.p64 = K.init_variables(self.spec, seed)
        self.params = b.upload(K.flatten(self.spec, self.p64))

    def oracle_logits(self, wav):
        c = self.cfg
        x = wav.astype(np.float64) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float64)
        kw = dict(num_mel_bins=c.num_mel_bins, sample_rate=c.sample_rate, lower_edge_hertz=c.lower_edge_hertz,
                  upper_edge_hertz=c.upper_edge_hertz)
        if c.feature_kind == L.TCR_FEATURE_MFCC:
            feat = O.mfcc(x, c.window_size_samples, c.window_stride_samples, num_mfccs=c.num_mfccs, **kw)
        else:
            feat = O.log_mel_spectrogram(x, c.window_size_samples, c.window_stride_samples, magnitude_squared=False, **kw)
        return K.forward(self.spec, self.p64, feat)


@pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])
@pytest.mark.parametrize("case", ["49x40", "98x40"])
def test_cuda_wav_forward_matches_features_and_oracle(cuda, arch, case):
    """fp32 and int16 clips: the forward from wav equals the forward on tcr_dscnn_mfcc_forward's features bit for bit, and the fp64
    front-end + oracle within 1e-4 (40 rows of each batch)."""
    ds = KwsDs(cuda, arch, FRONTENDS[case], 512, seed=5)
    try:
        for n, pcm in ((1, False), (3, True), (39, False), (512, True)):
            rows = np.unique(np.r_[np.arange(min(n, 32)), np.arange(max(0, n - 8), n)])
            check_parity(ds, clips(n, seed=n, pcm=pcm), rows)
    finally:
        ds.close()


def run_listener(b, arch, S, hop, K_, pushes, reset_at=(), pcm_every=3, seed=0, case="49x40"):
    """case: a FRONTENDS key or a dict of tcr_config front-end fields.  The launch check needs the CUDA build's profiler."""
    from listener_cases import Offline, random_chunk
    ds = KwsDs(b, arch, FRONTENDS[case] if isinstance(case, str) else case, S * K_, seed=seed)
    lis = DsListener(ds, S, hop, K_ * hop * ds.cfg.window_stride_samples)
    try:
        off = Offline(ds, S, hop)
        rng = np.random.default_rng(seed)
        for i in range(pushes):
            for r in (x for at, x in reset_at if at == i):
                lis.reset(r)
                for s in (range(S) if r == -1 else [r]):
                    off.reset(s)
            check_ds_push(ds, lis, off, random_chunk(rng, S, lis.chunk, pcm=(i % pcm_every == pcm_every - 1)))
        if b.name == "cuda":
            got = launched(b.lib, lambda: lis.push(np.zeros((S, lis.chunk), np.float32)))
            first = WIN_KERNEL[arch]
            assert got[first + ":win"] == 1 and first not in got, got
    finally:
        lis.close()
        ds.close()


@pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])
def test_cuda_listener_matches_the_cut_clips(cuda, arch):
    """13 streams x 3 windows at hop = T - 1 (fp32 and int16 pushes, reset of every stream and of the last one), and K = hop = 1."""
    run_listener(cuda, arch, S=13, hop=48, K_=3, pushes=4, reset_at=((2, -1), (3, 12)), pcm_every=2)
    run_listener(cuda, arch, S=7, hop=1, K_=1, pushes=5, pcm_every=2)


def test_cuda_kws_listeners_interleave_with_dscnn_and_tcresnet(cuda):
    """A trad_fpool3, a one_fstride4, a DS-CNN-S and a TC-ResNet listener pushed in turn: each keeps its own state and matches
    its own model."""
    from listener_cases import Listener, Offline, check_push, random_chunk, variables
    from tcr_harness import Engine
    eng = Engine(cuda, max_batch=4, dropout_keep_prob=1.0)
    tl = Listener(eng, 2, 2, 2 * 2 * eng.cfg.window_stride_samples)
    dss = [KwsDs(cuda, "trad_fpool3", FRONTENDS["49x40"], 6, seed=1), KwsDs(cuda, "one_fstride4", FRONTENDS["49x40"], 6, seed=2),
           Ds(cuda, "S", FRONTENDS["49x40"], 6, seed=3)]
    lis = [DsListener(d, 2, 3, 3 * 3 * d.cfg.window_stride_samples) for d in dss]
    try:
        p_h, m_h = variables(eng, 5)
        p, m = cuda.upload(p_h), cuda.upload(m_h)
        t_off, offs = Offline(eng, 2, 2), [Offline(d, 2, 3) for d in dss]
        rng = np.random.default_rng(3)
        for i in range(4):
            check_push(eng, tl, t_off, random_chunk(rng, 2, tl.chunk, pcm=i == 1), p_h, p, m_h, m)
            for d, l, o in zip(dss, lis, offs):
                check_ds_push(d, l, o, random_chunk(rng, 2, l.chunk, pcm=i == 2))
    finally:
        tl.close()
        for l in lis:
            l.close()
        for d in dss:
            d.close()
        eng.close()


def _flags(arch):
    return ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
            f"--window_size_ms 40 --window_stride_ms 20", f"KWSModel --architecture {arch}")


@pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])
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
    spec = K.build_spec(arch, 49, 40, 12)
    values = {k: v.astype(np.float32) for k, v in K.init_variables(spec, 2).items()}
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


@pytest.mark.parametrize("arch", ["trad_fpool3", "one_fstride4"])
def test_evaluate_audio_counts_the_oracles_predictions(tmp_path, arch):
    """The recipe's evaluation flags (--batch_size 3, --valid_type once) on a small on-disk split and a TF-V2 bundle of seeded
    weights under the bare names: the confusion matrix and accuracy equal the fp64 oracle's arg-max counts, total_loss is
    CE + 1e-4 * sum(w^2) / 2 and model_loss CE; --use_ema scores with the /ExponentialMovingAverage shadows."""
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper
    from tcresnet_b200.runtime import Session
    flags, model = _flags(arch)
    make_split(tmp_path, "valid", per_label=3, seed=2)
    spec = K.build_spec(arch, 49, 40, 12)
    values = {k: v.astype(np.float32) for k, v in K.init_variables(spec, 11).items()}
    shadows = {k: v.astype(np.float32) for k, v in K.init_variables(spec, 12).items()}
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
            ref = K.forward(spec, w64, O.mfcc(wav[..., 0].astype(np.float64), 640, 320, num_mfccs=40))
            top2 = np.sort(ref, axis=1)[:, -2:]
            assert (top2[:, 1] - top2[:, 0]).min() > 1e-4 * np.abs(ref).max()
            np.add.at(cm, (hot.argmax(1), ref.argmax(1)), 1)
            logp = ref - ref.max(1, keepdims=True)
            logp -= np.log(np.exp(logp).sum(1, keepdims=True))
            ces.append(-(hot * logp).sum(1).mean())
        return cm, float(np.mean(ces)), 1e-4 * K.l2_loss(w64)

    for extra, weights in (("", values), ("--use_ema", shadows)):
        results = evaluate_audio.main(args(extra))
        assert len(results) == 1
        got = results[0]
        cm, ce, l2 = oracle(weights)
        assert np.array_equal(np.asarray(got["confusion_matrix"]), cm), extra
        assert got["accuracy"] == np.trace(cm) / cm.sum()
        assert abs(got["total_loss"] - (ce + l2)) <= 1e-5 * abs(ce + l2), (got["total_loss"], ce, l2)
