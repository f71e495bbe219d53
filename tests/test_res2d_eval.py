"""The 2-D ablations of TC-ResNet8 on the GPU (ResNet2D8 / ResNet2D8Pool on the DS-CNN handle): each layer and the logits against
the fp64 oracle (res2d_oracle) with the kernels each layer launches, batch invariance, the wav input paths and the listener
against the forward on features / cut clips bit for bit, the evaluation counts, the deployable and streaming models,
listen_audio.py and evaluate_audio.py end to end."""
import ctypes as C
import shlex

import numpy as np
import pytest

from oracle import res2d_oracle as R
from oracle import tcr_oracle as O
from tcr_harness import launched
from test_dscnn import features
from test_dscnn_eval import FRONTENDS, Ds, check_parity, clips
from test_dscnn_listener import DsListener, check_ds_push
from test_res2d import GEOMETRY, Res2dNet, check_net, create

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L

pytestmark = pytest.mark.gpu

KERNELS = [["res2d_conv0"], ["res2d_block"], ["res2d_block"], ["res2d_block"]]


@pytest.fixture(scope="module")
def cuda():
    from tcr_harness import TorchBackend
    return TorchBackend()


def check_layers(net, feat, rows=None):
    """test_res2d.check_net on the GPU (the oracle on `rows`), with the kernel each layer launches (the launch profiler's counts)."""
    seen = {}
    orig = net.layer_output

    def layer_output(f, k):
        got = {}
        counts = launched(net.lib, lambda: got.setdefault("a", orig(f, k)))
        new = counts - seen["prev"] if "prev" in seen else counts
        assert sorted(new) == KERNELS[k - 1] and all(v == 1 for v in new.values()), (k, counts)
        seen["prev"] = counts
        return got["a"]
    net.layer_output = layer_output
    try:
        errs, logits = check_net(net, feat, rows=rows)
    finally:
        net.layer_output = orig
    assert launched(net.lib, lambda: net.forward(feat)) == {"res2d_conv0": 1, "res2d_block": 3, "res2d_head": 1}
    return errs, logits


@pytest.mark.parametrize("wm", [0.5, 1.0, 2.5])
@pytest.mark.parametrize("model,T,Fq", GEOMETRY)
def test_cuda_layers_and_logits_match_the_oracle(cuda, model, T, Fq, wm):
    """n = 1, 3 and 39 at every geometry row and width, and n = 512 = max_batch at 98 x 40 (MFCC statistics there).  The logits of an
    utterance are the same bits in any batch: permuted, and on a handle with another max_batch."""
    big = Res2dNet(cuda, model, T, Fq, 512, seed=1, wm=wm)
    small = Res2dNet(cuda, model, T, Fq, 39, seed=1, wm=wm)
    try:
        for n in (1, 3, 39) + ((512,) if (T, Fq) == (98, 40) else ()):
            feat = features("mfcc" if (T, Fq) == (98, 40) else "randn", n, T, Fq, seed=n)
            check_layers(big, feat)
            if n == 39:
                ref, _ = big.forward(feat)
                perm = np.random.RandomState(n).permutation(n)
                assert np.array_equal(big.forward(np.ascontiguousarray(feat[perm]))[0], ref[perm])
                assert np.array_equal(small.forward(feat)[0], ref)
    finally:
        big.close()
        small.close()


@pytest.mark.parametrize("model", ["ResNet2D8", "ResNet2D8Pool"])
def test_cuda_many_tiles_per_sm(cuda, model):
    """A batch whose block-kernel tile count exceeds 2 x the SM count many times over (n = 3,000 at 98 x 40), layer by layer on 64
    rows and bit-identical to the same utterances in a batch of 64."""
    import torch
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n = 3000
    net = Res2dNet(cuda, model, 98, 40, n, seed=4)
    small = Res2dNet(cuda, model, 98, 40, 64, seed=4)
    try:
        assert n > 2 * sms
        feat = np.random.RandomState(9).randn(n, 98, 40).astype(np.float32)
        logits, _ = net.forward(feat)
        rows = np.r_[0:32, n - 32:n]
        assert np.array_equal(small.forward(np.ascontiguousarray(feat[rows]))[0], logits[rows])
        ref = R.forward(net.spec, net.p, feat[rows].astype(np.float64))
        assert np.abs(logits[rows] - ref).max() <= 1e-4 * np.abs(ref).max()
        check_layers(small, np.ascontiguousarray(feat[rows]))
    finally:
        net.close()
        small.close()


class Res2dDs(Ds):
    """test_dscnn_eval.Ds on a 2-D ablation handle: the front-end, res2d_oracle's seeded variables and its fp64 logits."""

    def __init__(self, b, model, frontend, max_batch, seed=0, classes=12, wm=1.0):
        self.b, self.lib, self.model = b, b.lib, model
        c = L.TcrConfig()
        L.check(self.lib, self.lib.tcr_config_default(C.byref(c)), "tcr_config_default")
        for k, v in frontend.items():
            setattr(c, k, v)
        c.num_classes = classes
        self.cfg = c
        T = 1 + (c.clip_samples - c.window_size_samples) // c.window_stride_samples
        F = c.num_mfccs if c.feature_kind == L.TCR_FEATURE_MFCC else c.num_mel_bins
        self.T, self.F, self.classes, self.size = T, F, classes, R.CODES[model]
        self.info = type("Info", (), dict(frames=T, features=F))
        rc, self.h = create(self.lib, model, T, F, max_batch, classes, wm)
        L.check(self.lib, rc, "tcr_dscnn_create")
        L.check(self.lib, self.lib.tcr_dscnn_set_frontend(self.h, C.byref(c)), "tcr_dscnn_set_frontend")
        self.spec = R.build_spec(model, T, F, classes, wm)
        self.p64 = R.init_variables(self.spec, seed)
        self.params = b.upload(R.flatten(self.spec, self.p64))

    def features64(self, wav):
        c = self.cfg
        x = wav.astype(np.float64) / 32768.0 if wav.dtype == np.int16 else wav.astype(np.float64)
        kw = dict(num_mel_bins=c.num_mel_bins, sample_rate=c.sample_rate, lower_edge_hertz=c.lower_edge_hertz,
                  upper_edge_hertz=c.upper_edge_hertz)
        if c.feature_kind == L.TCR_FEATURE_MFCC:
            return O.mfcc(x, c.window_size_samples, c.window_stride_samples, num_mfccs=c.num_mfccs, **kw)
        return O.log_mel_spectrogram(x, c.window_size_samples, c.window_stride_samples, magnitude_squared=False, **kw)

    def oracle_logits(self, wav):
        return R.forward(self.spec, self.p64, self.features64(wav))


LOGMEL128 = dict(feature_kind=L.TCR_FEATURE_LOG_MEL, num_mel_bins=128, window_size_samples=480, window_stride_samples=160)


@pytest.mark.parametrize("model", ["ResNet2D8", "ResNet2D8Pool"])
@pytest.mark.parametrize("case", ["98x40", "49x10", "logmel128"])
def test_cuda_wav_forward_matches_features_and_oracle(cuda, model, case):
    """fp32 and int16 clips: the forward from wav equals the forward on tcr_dscnn_mfcc_forward's features bit for bit, and the fp64
    front-end + oracle within 1e-4 (40 rows of each batch)."""
    ds = Res2dDs(cuda, model, LOGMEL128 if case == "logmel128" else FRONTENDS[case], 512, seed=5)
    try:
        for n, pcm in ((1, False), (3, True), (39, False), (512, True)):
            rows = np.unique(np.r_[np.arange(min(n, 32)), np.arange(max(0, n - 8), n)])
            check_parity(ds, clips(n, seed=n, pcm=pcm), rows)
    finally:
        ds.close()


@pytest.mark.parametrize("model", ["ResNet2D8", "ResNet2D8Pool"])
def test_cuda_eval_counts_equal_the_oracles_predictions(cuda, model):
    """tcr_dscnn_eval_accumulate on the forward's softmax: the confusion matrix is the oracle's arg-max against the labels."""
    import torch
    ds = Res2dDs(cuda, model, FRONTENDS["98x40"], 64, seed=6)
    try:
        n = 64
        wav = clips(n, seed=21)
        logits, probs = ds.wav_forward(wav)
        ref = ds.oracle_logits(wav)
        top2 = np.sort(ref, axis=1)[:, -2:]
        assert (top2[:, 1] - top2[:, 0]).min() > 2 * np.abs(logits - ref).max()
        labels = np.random.RandomState(3).randint(0, 12, n)
        hot = np.eye(12, dtype=np.float32)[labels]
        counts = torch.zeros(12 * 12 + 2, dtype=torch.int64, device="cuda")
        d_probs, d_hot = cuda.upload(probs), cuda.upload(hot)
        L.check(ds.lib, ds.lib.tcr_dscnn_eval_accumulate(ds.h, cuda.ptr(d_probs), cuda.ptr(d_hot), n, 5, counts.data_ptr(),
                                                         cuda.stream), "tcr_dscnn_eval_accumulate")
        got = counts.cpu().numpy()
        cm = np.zeros((12, 12), np.int64)
        np.add.at(cm, (labels, ref.argmax(1)), 1)
        assert np.array_equal(got[:144].reshape(12, 12), cm)
    finally:
        ds.close()


def run_listener(b, model, S, hop, K_, pushes, reset_at=(), pcm_every=3, seed=0, case="98x40", wm=1.0):
    """case: a FRONTENDS key or a dict of tcr_config front-end fields; wm: the width multiplier.  The launch check needs the CUDA
    build's profiler."""
    from listener_cases import Offline, random_chunk
    ds = Res2dDs(b, model, FRONTENDS[case] if isinstance(case, str) else case, S * K_, seed=seed, wm=wm)
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
            assert got["res2d_conv0:win"] == 1 and "res2d_conv0" not in got, got
    finally:
        lis.close()
        ds.close()


@pytest.mark.parametrize("model", ["ResNet2D8", "ResNet2D8Pool"])
def test_cuda_listener_matches_the_cut_clips(cuda, model):
    """13 streams x 3 windows at hop = T - 1 (fp32 and int16 pushes, a reset of every stream and of the last one), K = hop = 1, and
    10 MFCCs (odd-width history rows)."""
    run_listener(cuda, model, S=13, hop=97, K_=3, pushes=4, reset_at=((2, -1), (3, 12)), pcm_every=2)
    run_listener(cuda, model, S=7, hop=1, K_=1, pushes=5, pcm_every=2)
    run_listener(cuda, model, S=3, hop=5, K_=2, pushes=3, case="49x10")


def test_cuda_res2d_listeners_interleave_with_dscnn_kws_and_tcresnet(cuda):
    """A ResNet2D8, a ResNet2D8Pool, a DS-CNN-S, a trad_fpool3 and a TC-ResNet listener pushed in turn: each keeps its own state and
    matches its own model."""
    from listener_cases import Listener, Offline, check_push, random_chunk, variables
    from tcr_harness import Engine
    from test_kws_eval import KwsDs
    eng = Engine(cuda, max_batch=4, dropout_keep_prob=1.0)
    tl = Listener(eng, 2, 2, 2 * 2 * eng.cfg.window_stride_samples)
    dss = [Res2dDs(cuda, "ResNet2D8", FRONTENDS["49x40"], 6, seed=1), Res2dDs(cuda, "ResNet2D8Pool", FRONTENDS["49x40"], 6, seed=2),
           Ds(cuda, "S", FRONTENDS["49x40"], 6, seed=3), KwsDs(cuda, "trad_fpool3", FRONTENDS["49x40"], 6, seed=4)]
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


FLAGS = ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
         "--window_size_ms 30 --window_stride_ms 10")


@pytest.mark.parametrize("model", ["ResNet2D8Model", "ResNet2D8PoolModel"])
def test_deployed_and_streaming_models_and_listen_audio(cuda, tmp_path, model):
    """build_deployable_model: eager calls then graph replay, each equal to forward_input on the clip; build_streaming_model pushes
    equal to forward_input on the cut clips; listen_audio.py on a checkpoint writes one .npy and .csv per file, the softmaxes of the
    forward on its windows.  Width 0.5 through --width_multiplier."""
    import torch
    from listener_cases import Offline, random_chunk
    from test_listener import _write_wav
    from tcresnet_b200 import evaluate_audio, listen_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.factory import audio_nets
    tail = f"{model} --width_multiplier 0.5"
    args = evaluate_audio.parse_arguments(shlex.split(f"--dataset_path synthetic:8 --dataset_split_name valid --checkpoint_path x "
                                                      f"--batch_size 1 --augmentation_method anchored_slice_or_pad {FLAGS} {tail}"))
    m = getattr(audio_nets, model)(args, None)
    _, dep = m.build_deployable_model(include_preprocess=True)
    assert m.engine.table[0]["shape"] == (3, 3, 1, R.channels(40, 0.5)[0])
    for i in range(4):
        x = clips(1, seed=10 + i)
        assert np.array_equal(dep(x), m.engine.forward_input(torch.from_numpy(x).cuda(), m.params)[1].cpu().numpy()), i
    assert dep._graph is not None
    sm = m.build_streaming_model(streams=3, hop_ms=40, chunk_ms=120)
    off = Offline(type("E", (), dict(cfg=sm.engine.cfg, info=sm.engine.info)), 3, 4)
    rng = np.random.default_rng(0)
    for i in range(4):
        x = random_chunk(rng, 3, sm.chunk_samples, pcm=i == 2)
        got = sm(x)
        cut = off.push(x).reshape(9, -1)
        ref = sm.engine.forward_input(torch.from_numpy(cut).cuda(), m.params)[1].cpu().numpy().reshape(3, 3, -1)
        assert np.array_equal(got, ref), i
    sm.listener.close()
    scope = model[:-len("Model")]
    spec = R.build_spec(scope, 98, 40, 12, 0.5)
    values = {k: v.astype(np.float32) for k, v in R.init_variables(spec, 2).items()}
    path = ckpt.save(tmp_path / "run", model, 100, values, fmt="tf")
    wav = rng.integers(-20000, 20000, 12000).astype(np.int16)
    _write_wav(tmp_path / "a.wav", wav)
    out = tmp_path / "out"
    la = listen_audio.parse_arguments(shlex.split(f"--checkpoint_path {path} --hop_ms 40 --chunk_ms 120 --output_dir {out} "
                                                  f"{FLAGS} {tail} {tmp_path / 'a.wav'}"))
    results = listen_audio.listen(la)
    assert len(results) == 1
    assert np.array_equal(np.load(out / "a.npy"), results[0]) and (out / "a.csv").is_file()
    assert results[0].shape == (-(-12000 // 640), 12) and np.allclose(results[0].sum(1), 1, atol=1e-5)
    m.set_variables(values)
    off = Offline(type("E", (), dict(cfg=m.engine.cfg, info=m.engine.info)), 1, 4)
    pushes = -(-results[0].shape[0] // 3)
    stream = np.zeros((1, pushes * 1920), np.float32)
    stream[0, :12000] = wav.astype(np.float32) / 32768.0
    cut = np.concatenate([off.push(stream[:, p * 1920:(p + 1) * 1920]) for p in range(pushes)], axis=1)[0][:results[0].shape[0]]
    ref = np.concatenate([sm.engine.forward_input(torch.from_numpy(np.ascontiguousarray(cut[i:i + 3])).cuda(), m.params)[1].cpu().numpy()
                          for i in range(0, cut.shape[0], 3)])
    assert np.array_equal(results[0], ref)
    sm.engine.close()
    m.engine.close()


@pytest.mark.parametrize("model", ["ResNet2D8Model", "ResNet2D8PoolModel"])
def test_evaluate_audio_counts_the_oracles_predictions(tmp_path, model):
    """The recipe's evaluation flags (--weight_decay 0.001, --batch_size 3, --valid_type once) on a small on-disk split and a TF-V2
    bundle of seeded weights: the confusion matrix and accuracy equal the fp64 oracle's arg-max counts, total_loss is CE plus
    0.001 * sum(w^2) / 2 over the non-BatchNorm variables (fc2 included) and model_loss CE; --use_ema scores with the
    /ExponentialMovingAverage shadows of the trainable variables."""
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper
    from tcresnet_b200.runtime import Session
    make_split(tmp_path, "valid", per_label=3, seed=2)
    scope = model[:-len("Model")]
    spec = R.build_spec(scope, 98, 40, 12)
    values = {k: v.astype(np.float32) for k, v in R.init_variables(spec, 11).items()}
    shadows = {k: v.astype(np.float32) for k, v in R.init_variables(spec, 12).items()}
    bundle = dict(values, **{k + "/ExponentialMovingAverage": v for k, v in shadows.items()})
    path = ckpt.save(tmp_path / "run", model, 1000, bundle, fmt="tf")

    def args(extra=""):
        return evaluate_audio.parse_arguments(shlex.split(
            f"--dataset_path {tmp_path} --dataset_split_name valid --checkpoint_path {path} --num_silent 6 "
            "--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 3 "
            f"--no-shuffle --valid_type once --no-save_best_keeper {extra} {FLAGS} {model} --weight_decay 0.001"))

    def oracle(weights):
        session = Session()
        ds = SingleLabelAudioDataWrapper(args(), session, "valid", False)
        ds.get_input_and_output_op()
        ds.setup_iterator(session, ds.placeholders, ds.data)
        cm, ces = np.zeros((12, 12)), []
        w64 = {k: np.asarray(v, np.float64) for k, v in weights.items()}
        for _ in range(ds.num_samples // 3):
            wav, hot = ds.next_batch()
            ref = R.forward(spec, w64, O.mfcc(wav[..., 0].astype(np.float64), 480, 160, num_mfccs=40))
            top2 = np.sort(ref, axis=1)[:, -2:]
            assert (top2[:, 1] - top2[:, 0]).min() > 1e-4 * np.abs(ref).max()
            np.add.at(cm, (hot.argmax(1), ref.argmax(1)), 1)
            logp = ref - ref.max(1, keepdims=True)
            logp -= np.log(np.exp(logp).sum(1, keepdims=True))
            ces.append(-(hot * logp).sum(1).mean())
        return cm, float(np.mean(ces)), R.l2_loss(spec, w64, 0.001)

    # --use_ema takes each trainable variable from its shadow; the BatchNorm moving statistics are not trainable and keep theirs
    ema = {k: (values if "/moving_" in k else shadows)[k] for k in values}
    for extra, weights in (("", values), ("--use_ema", ema)):
        results = evaluate_audio.main(args(extra))
        assert len(results) == 1
        got = results[0]
        cm, ce, l2 = oracle(weights)
        assert np.array_equal(np.asarray(got["confusion_matrix"]), cm), extra
        assert got["accuracy"] == np.trace(cm) / cm.sum()
        assert abs(got["total_loss"] - (ce + l2)) <= 1e-5 * abs(ce + l2), (got["total_loss"], ce, l2)
