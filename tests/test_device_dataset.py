"""--device_dataset: a split decoded once into device memory, every batch gathered and augmented there with draws made in the
kernel (tcr_dataset_batch, tcr_step_args::dataset).  Kernel logic against the NumPy restatement (tests/dataset_oracle.py) on the
CPU emulator; the sm_90a build, the trainer and the evaluator under -m gpu."""
import ctypes as C
import os
import shlex
import wave

import numpy as np
import pytest
from scipy import stats

import dataset_oracle as D
from oracle import augment_oracle as A
from oracle import tcr_oracle as O
from tcr_harness import Engine, NumpyBackend

import tcresnet_b200  # noqa: F401
from tcresnet_b200 import _lib as L
from tcresnet_b200.datasets import augmentation_factory as H
from tcresnet_b200.datasets import device_input_stage as S

CLIP = 16000
LABELS = ["down", "go", "left", "no", "off", "on", "right", "stop", "unknown", "up", "yes"]


def _write_wav(path, samples, channels=1):
    with wave.open(str(path), "wb") as w:
        w.setnchannels(channels)
        w.setsampwidth(2)
        w.setframerate(16000)
        w.writeframes(np.ascontiguousarray(samples, "<i2").tobytes())


def make_split(root, split, per_label=4, seed=0):
    """A seeded Speech Commands-like split: clips shorter and longer than 1 s, one stereo file, and a _background_noise_
    directory with one recording shorter than a clip."""
    rng = np.random.RandomState(seed)
    d = root / split
    for li, label in enumerate(LABELS):
        (d / label).mkdir(parents=True)
        for k in range(per_label):
            length = [CLIP, 9000, 21000, 15999][(li + k) % 4]
            x = rng.randint(-20000, 20000, length).astype(np.int16)
            if li == 0 and k == 0:
                _write_wav(d / label / f"{k:03d}.wav", np.stack([x, -x], 1), channels=2)
            else:
                _write_wav(d / label / f"{k:03d}.wav", x)
    noise = d / "_background_noise_"
    noise.mkdir()
    for j, length in enumerate([40000, 12000, 70000]):
        _write_wav(noise / f"noise{j}.wav", rng.randint(-30000, 30000, length).astype(np.int16))
    return root


def _args(root, split="train", extra=""):
    from tcresnet_b200 import train_audio
    return train_audio.parse_arguments(shlex.split(
        f"--dataset_path {root} --dataset_split_name {split} --output_name output/softmax --num_classes 12 --num_silent 5 "
        f"--preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 "
        f"--train_dir {root}/run --augmentation_method anchored_slice_or_pad_with_shift --batch_size 4 --boundaries 100000 "
        f"--max_step_from_restore 12 --lr_list 0.1 0.01 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100000 "
        f"--step_evaluation 100000 --step_save_summaries 100000 --step_save_first_n_summaries 0 --optimizer mom --momentum 0.9 "
        f"{extra} TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))


def _padded_background(arrays, clip=CLIP):
    bank = [np.pad(b, (0, clip - b.shape[0])) if b.shape[0] < clip else b for b in arrays]
    return np.concatenate(bank).astype(np.float32), [b.shape[0] for b in bank]


# ----------------------------------------------------------------------------------------------------- oracle statistics
def test_oracle_draw_statistics():
    n = 100_000
    bg_lengths = [40000, 23000, 70000, 16000, 61000, 30000]
    d = D.draws(99, 3, np.arange(n), CLIP, bg_lengths)
    assert d["shift"].min() >= -1600 and d["shift"].max() < 1600
    assert stats.chisquare(np.bincount(d["shift"] + 1600, minlength=3200)).pvalue > 1e-4
    assert stats.chisquare(np.bincount(d["recording"], minlength=6)).pvalue > 1e-4
    rate, sigma = d["mixed"].mean(), np.sqrt(0.8 * 0.2 / n)
    assert abs(rate - 0.8) < 4 * sigma
    v = d["volume"][d["mixed"]]
    assert v.dtype == np.float32 and v.min() >= 0 and v.max() < 0.1
    assert (d["volume"][~d["mixed"]] == 0).all()
    lengths = np.asarray(bg_lengths)
    assert (d["crop"] >= 0).all() and (d["crop"] <= lengths[d["recording"]] - CLIP).all()
    # a key is (seed, epoch, position): another epoch draws other numbers, the same key the same ones
    assert not np.array_equal(D.draws(99, 4, np.arange(64), CLIP, bg_lengths)["shift"], d["shift"][:64])
    assert np.array_equal(D.draws(99, 3, np.arange(10, 74), CLIP, bg_lengths)["shift"], d["shift"][10:74])


# ----------------------------------------------------------------------------------------------------- the batch kernel
def _desc(b, bank, table, order, background, bg_lengths, shift, mix, training, freq, vol):
    """TcrDataset over backend buffers; returns (desc, keep-alive list)."""
    clip_bytes = np.frombuffer(np.ascontiguousarray(table, S.DATASET_CLIP_DTYPE).tobytes(), np.uint8)
    bg_table = np.stack([np.cumsum(bg_lengths) - np.asarray(bg_lengths), np.asarray(bg_lengths)], 1).astype(np.int64).reshape(-1)
    keep = [b.upload(np.ascontiguousarray(bank, np.int16)), b.upload_bytes(clip_bytes),
            b.upload_bytes(np.frombuffer(np.ascontiguousarray(order, np.int32).tobytes(), np.uint8)),
            b.upload(background) if background is not None else None,
            b.upload_bytes(np.frombuffer(bg_table.tobytes(), np.uint8))]
    d = L.TcrDataset()
    d.samples, d.num_samples = b.ptr(keep[0]), len(bank)
    d.clips, d.num_clips = b.ptr(keep[1]), len(table)
    d.order, d.order_length = b.ptr(keep[2]), len(order)
    d.background, d.background_samples = b.ptr(keep[3]), 0 if background is None else len(background)
    d.background_table, d.num_background = b.ptr(keep[4]), len(bg_lengths)
    d.shift, d.mix, d.is_training = int(shift), int(mix), int(training)
    d.background_frequency, d.background_max_volume = freq, vol
    return d, keep


def _dataset_batch(eng, desc, position, epoch, seed, n):
    b = eng.b
    wav, hot = b.empty(n, CLIP), b.empty(n, eng.cfg.num_classes)
    L.check(eng.lib, eng.lib.tcr_dataset_batch(eng.h, C.byref(desc), position, epoch, seed, n, b.ptr(wav), b.ptr(hot), b.stream),
            "tcr_dataset_batch")
    b.sync()
    return b.download(wav), b.download(hot)


def _synthetic_bank(rng, num_clips):
    lengths = rng.randint(1, CLIP + 1, num_clips)
    lengths[::7] = 0                                                          # silent samples
    lengths[1::7] = CLIP                                                      # cropped at decode
    lengths[2::7] = 9000                                                      # short
    table = np.zeros(num_clips, S.DATASET_CLIP_DTYPE)
    table["offset"], table["length"], table["label"] = np.cumsum(lengths) - lengths, lengths, rng.randint(0, 12, num_clips)
    bank = rng.randint(-32768, 32768, int(lengths.sum())).astype(np.int16)
    return bank, table


def _extreme_shift_positions(seed, epoch, count):
    s = D.draws(seed, epoch, np.arange(count), CLIP, [])["shift"]
    return int(np.argmax(s == 1599)), int(np.argmax(s == -1600))


def _check_batches(backend, num_clips, n, seed=5):
    rng = np.random.RandomState(seed)
    bank, table = _synthetic_bank(rng, num_clips)
    background, bg_lengths = _padded_background([rng.uniform(-1, 1, k).astype(np.float32) for k in (40000, 12000, 70000)])
    count = 40_000
    order = rng.randint(0, num_clips, count).astype(np.int32)
    hi, lo = _extreme_shift_positions(seed, 2, count)
    eng = Engine(backend, max_batch=n)
    for freq, vol in ((0.8, 0.1), (1.0, 1.0)):                               # volume up to 1: the clip to [-1, 1] acts
        desc, keep = _desc(backend, bank, table, order, background, bg_lengths, True, True, True, freq, vol)
        for position in (0, max(0, hi - n // 2), max(0, lo - n // 2)):
            got, hot = _dataset_batch(eng, desc, position, 2, seed, n)
            ref, ref_hot = D.batch(bank, table, order, position, n, seed, 2, CLIP, 12, background, bg_lengths,
                                   background_frequency=freq, background_max_volume=vol)
            assert np.array_equal(got, ref), np.abs(got - ref).max()
            assert np.array_equal(hot, ref_hot)
    positions = set(range(0, n)) | set(range(max(0, hi - n // 2), max(0, hi - n // 2) + n))
    assert hi in positions and table["length"][order[:n]].min() == 0
    # evaluation settings: no shift, volume 0 -> the decoded clip, zero-padded
    desc, keep = _desc(backend, bank, table, order, background, bg_lengths, False, True, False, 0.8, 0.1)
    got, hot = _dataset_batch(eng, desc, 0, 0, seed, n)
    for i in range(n):
        c = table[order[i]]
        ref = np.zeros(CLIP, np.float32)
        ref[:c["length"]] = bank[c["offset"]:c["offset"] + c["length"]].astype(np.float32) / np.float32(32768.0)
        assert np.array_equal(got[i], ref)
    eng.close()


def test_emulated_dataset_batch_is_bit_exact():
    _check_batches(NumpyBackend(), 40, 6)


def test_emulated_dataset_batch_stays_inside_the_banks():
    """Order entries outside the table, clips outside the bank and labels outside the classes read nothing out of bounds."""
    b = NumpyBackend()
    rng = np.random.RandomState(1)
    bank, table = _synthetic_bank(rng, 6)
    table["length"][:] = 9000
    table["offset"][3] = len(bank) - 100                                      # runs past the end of the bank: 100 samples read
    table["offset"][4] = len(bank) + 5                                        # entirely outside: silent
    table["label"][5] = 40                                                    # no class: an all-zero one-hot row
    order = np.array([-1, 6, 3, 4, 5], np.int32)
    background, bg_lengths = _padded_background([rng.uniform(-1, 1, 20000).astype(np.float32)])
    desc, keep = _desc(b, bank, table, order, background, bg_lengths, False, True, False, 0.8, 0.1)
    eng = Engine(b, max_batch=5)
    got, hot = _dataset_batch(eng, desc, 0, 0, 1, 5)
    assert (got[[0, 1, 3]] == 0).all() and (hot[[0, 1, 4]] == 0).all()
    assert np.array_equal(got[2, :100], bank[-100:].astype(np.float32) / np.float32(32768.0)) and (got[2, 100:] == 0).all()
    with pytest.raises(L.TcrError, match="outside the order"):
        _dataset_batch(eng, desc, 1, 0, 1, 5)
    eng.close()


def test_emulated_batch_equals_the_host_path_decode_in_evaluation(tmp_path):
    """Evaluation settings on a bank decoded from wav files == load_wav_file's pad / crop, file by file."""
    make_split(tmp_path, "valid", per_label=1)
    files = sorted(str(p) for p in (tmp_path / "valid").glob("*/*.wav") if "_background_noise_" not in str(p)) + [""]
    bank, table = S.decode_clip_bank(files, list(range(len(files))) , CLIP, num_threads=3)
    table["label"] %= 12
    b = NumpyBackend()
    order = np.arange(len(files), dtype=np.int32)
    desc, keep = _desc(b, bank, table, order, None, [], False, False, False, 0.0, 0.0)
    eng = Engine(b, max_batch=len(files))
    got, _ = _dataset_batch(eng, desc, 0, 0, 0, len(files))
    for i, f in enumerate(files):
        ref = np.zeros(CLIP, np.float32) if f == "" else H.load_wav_file(f, CLIP)
        assert np.array_equal(got[i], ref), f
    eng.close()


def test_emulated_step_on_the_dataset_equals_the_step_on_the_oracle_batch():
    b = NumpyBackend()
    rng = np.random.RandomState(8)
    bank, table = _synthetic_bank(rng, 12)
    background, bg_lengths = _padded_background([rng.uniform(-1, 1, 30000).astype(np.float32)])
    order = rng.permutation(12).astype(np.int32)
    n, position, epoch, seed = 3, 4, 1, 77
    eng = Engine(b, max_batch=n)
    spec = O.build_spec("TCResNet8", 1.0, 49)
    pv, mv = O.init_variables(spec, 3)
    params, moving = O.flatten_vars(spec, pv).astype(np.float32), O.flatten_moving(spec, mv).astype(np.float32)
    wav, hot = D.batch(bank, table, order, position, n, seed, epoch, CLIP, 12, background, bg_lengths)
    ref = eng.train_step(wav, hot, params, np.zeros_like(params), moving, seed=4)
    desc, keep = _desc(b, bank, table, order, background, bg_lengths, True, True, True, 0.8, 0.1)
    p, sl, mv_, losses = params.copy(), np.zeros_like(params), moving.copy(), np.zeros(2, np.float32)
    a = L.TcrStepArgs()
    a.n, a.params, a.slots, a.moving, a.losses = n, p.ctypes.data, sl.ctypes.data, mv_.ctypes.data, losses.ctypes.data
    a.learning_rate, a.momentum, a.weight_decay, a.dropout_seed, a.apply_update = 0.1, 0.9, 1e-3, 4, 1
    a.dataset, a.dataset_position, a.dataset_epoch, a.dataset_seed = C.addressof(desc), position, epoch, seed
    L.check(eng.lib, eng.lib.tcr_train_step(eng.h, C.byref(a), None), "tcr_train_step")
    assert np.array_equal(p, ref["params"]) and np.array_equal(sl, ref["slots"]) and np.array_equal(mv_, ref["moving"])
    assert np.array_equal(losses, ref["losses"])
    a.dataset_position = 10                                                   # rows [10, 13) of an order of 12
    with pytest.raises(L.TcrError, match="outside the order"):
        L.check(eng.lib, eng.lib.tcr_train_step(eng.h, C.byref(a), None), "tcr_train_step")
    eng.close()


# ----------------------------------------------------------------------------------------------------- host logic
class _OrderSink:
    def __init__(self):
        self.orders = []

    def upload_order(self, order):
        self.orders.append(np.array(order))


def _wrapper(args, rank=0, world=1):
    from tcresnet_b200.datasets.audio_data_wrapper import SingleLabelAudioDataWrapper
    from tcresnet_b200.runtime import Session
    w = SingleLabelAudioDataWrapper(args, Session(), "train", True)
    w.rank, w.world = rank, world                  # the shuffle order does not depend on them: the wrapper stays at epoch 0
    return w


def test_bank_file_list_labels_and_samples_are_the_host_paths(tmp_path):
    make_split(tmp_path, "train")
    host = _wrapper(_args(tmp_path))
    dev = _wrapper(_args(tmp_path, extra="--device_dataset --num_threads 3"))
    assert dev.filenames == host.filenames and dev.labels == host.labels and dev.label_names == host.label_names
    table, bank = dev._bank_table, dev._bank
    assert table["label"].tolist() == host.labels
    for i, f in enumerate(host.filenames):
        x = np.zeros(0, np.int16) if f == "" else H.read_wav_pcm16(f)[:CLIP]
        assert table["length"][i] == x.shape[0] and np.array_equal(bank[table["offset"][i]:][:x.shape[0]], x)
    assert (table["length"] == 0).sum() == 5 and table["length"].max() == CLIP
    stereo = [i for i, f in enumerate(host.filenames) if f.endswith("down/000.wav")][0]
    with wave.open(host.filenames[stereo]) as w:
        assert w.getnchannels() == 2
    assert len(dev.background_data) == 3 and min(b.shape[0] for b in dev.background_data) < CLIP


@pytest.mark.parametrize("world", [1, 2])
def test_positions_follow_the_host_paths_order(tmp_path, world):
    """Over two epochs the device path reads, for every rank, exactly the sample indices _take_indices gives the host path; the
    draws of rank r's rows are those of rows [r n, (r + 1) n) of a one-GPU run with the global batch."""
    make_split(tmp_path, "train")
    n = 4
    total = len(_wrapper(_args(tmp_path)).filenames)
    steps = 2 * (total // (n * world)) + 1
    for rank in range(world):
        host = _wrapper(_args(tmp_path), rank, world)
        dev = _wrapper(_args(tmp_path), rank, world)
        dev.device_data = sink = _OrderSink()
        one = _wrapper(_args(tmp_path, extra=f"--batch_size {n * world}"))
        one.device_data = one_sink = _OrderSink()
        epochs = set()
        for _ in range(steps):
            idx = host._take_indices()
            pos, epoch = dev.next_device_rows()
            gpos, gepoch = one.next_device_rows()
            epochs.add(epoch)
            assert np.array_equal(sink.orders[-1][pos:pos + n], idx)
            assert pos == gpos + rank * n and epoch == gepoch and np.array_equal(sink.orders[-1], one_sink.orders[-1])
            mine = D.draws(1234, epoch, np.arange(pos, pos + n), CLIP, [40000, 16000, 70000])
            glob = D.draws(1234, gepoch, np.arange(gpos, gpos + n * world), CLIP, [40000, 16000, 70000])
            for k in mine:
                assert np.array_equal(mine[k], glob[k][rank * n:(rank + 1) * n])
        assert len(epochs) == 3 and len(sink.orders) == 3                   # one upload per epoch


def test_synthetic_data_is_refused(tmp_path):
    from tcresnet_b200 import train_audio
    args = train_audio.parse_arguments(shlex.split(
        "--dataset_path synthetic:64 --dataset_split_name train --output_name output/softmax --num_classes 12 "
        f"--augmentation_method anchored_slice_or_pad --preprocess_method mfcc --train_dir {tmp_path} --device_dataset TCResNet8Model"))
    with pytest.raises(ValueError, match="--device_dataset"):
        _wrapper(args)


# ----------------------------------------------------------------------------------------------------- on the H100
@pytest.mark.gpu
def test_cuda_dataset_batch_is_bit_exact():
    from tcr_harness import TorchBackend
    _check_batches(TorchBackend(), 4096, 512)


def _oracle_replay(model_args, host, steps, lr_schedule):
    """The steps of a --device_dataset run driven through Engine.train_step on oracle-built batches, from the same start."""
    import torch
    from tcresnet_b200.engine import Engine as PublicEngine
    a = model_args
    eng = PublicEngine(model="TCResNet8", num_classes=12, window_size_ms=a.window_size_ms, window_stride_ms=a.window_stride_ms,
                       max_batch=a.batch_size, dropout_keep_prob=a.dropout_keep_prob)
    params, slots, moving = eng.new_variables(seed=getattr(a, "seed", 0) or 0)
    bank, table = S.decode_clip_bank(host.filenames, host.labels, CLIP, 2)
    background, bg_lengths = _padded_background(host.background_data)
    labels = []
    for g in range(steps):
        idx = host._take_indices()
        pos = host._cursor - a.batch_size
        wav, hot = D.batch(bank, table, host._order, pos, a.batch_size, 1234, host._epoch, CLIP, 12, background, bg_lengths)
        assert np.array_equal(np.argmax(hot, 1), np.asarray(host.labels)[idx])
        labels.append(np.argmax(hot, 1))
        eng.train_step(torch.from_numpy(wav).cuda(), torch.from_numpy(hot).cuda(), params, slots, moving, lr_schedule(g), 0.9,
                       a.weight_decay, dropout_seed=g)
    torch.cuda.synchronize()
    return params.cpu().numpy(), slots.cpu().numpy(), moving.cpu().numpy(), labels


@pytest.mark.gpu
@pytest.mark.parametrize("resident", [None, "0"])
def test_train_audio_with_the_device_dataset_matches_the_oracle_batches(tmp_path, monkeypatch, resident):
    from tcresnet_b200 import train_audio
    if resident is not None:
        monkeypatch.setenv("TCR_RESIDENT", resident)
    make_split(tmp_path, "train", per_label=6)
    args = _args(tmp_path, extra="--device_dataset --batch_size 16")
    trainer = train_audio.train(args)
    model = trainer.model
    model.flush_feed()
    assert model.global_step == 12 and np.isfinite(model._feed_last[1]) and model._feed_last[0] == 12
    params, slots, moving, _ = _oracle_replay(args, _wrapper(_args(tmp_path, extra="--batch_size 16")), 12, model.lr_schedule)
    assert np.array_equal(model.params.cpu().numpy(), params)
    assert np.array_equal(model.slots.cpu().numpy(), slots)
    assert np.array_equal(model.moving.cpu().numpy(), moving)


@pytest.mark.gpu
def test_evaluate_audio_with_and_without_the_device_dataset(tmp_path):
    from tcresnet_b200 import evaluate_audio, train_audio
    make_split(tmp_path, "train", per_label=3)
    make_split(tmp_path, "valid", per_label=3, seed=1)
    train_audio.train(_args(tmp_path, extra="--device_dataset"))
    results = {}
    for extra in ("", "--device_dataset"):
        e = evaluate_audio.parse_arguments(shlex.split(
            f"--dataset_path {tmp_path} --dataset_split_name valid --output_name output/softmax --num_classes 12 --num_silent 5 "
            f"--checkpoint_path {tmp_path}/run --augmentation_method anchored_slice_or_pad --preprocess_method mfcc --num_mfccs 40 "
            f"--clip_duration_ms 1000 --window_size_ms 40 --window_stride_ms 20 --background_frequency 0.0 "
            f"--background_max_volume 0.0 --batch_size 4 --no-shuffle --valid_type once --no-save_best_keeper {extra} "
            f"TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
        results[extra] = evaluate_audio.main(e)[0]
    host, dev = results[""], results["--device_dataset"]
    assert set(host) == set(dev)
    for k in host:
        assert np.array_equal(np.asarray(host[k]), np.asarray(dev[k])), k


@pytest.mark.gpu
def test_data_parallel_device_dataset_keeps_the_replicas_identical(tmp_path):
    """train_audio --data_parallel --device_dataset under torchrun on 2 GPUs, 12 steps: parameters, slots and moving statistics
    bit-identical on both ranks, and rank r read rows [r n, (r + 1) n) of the host path's global batch (tests/dist_device_dataset_worker.py)."""
    import subprocess
    import sys
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    make_split(tmp_path, "train", per_label=36)                               # 401 samples: 12 steps of 2 x 16 in one epoch
    worker = os.path.join(os.path.dirname(os.path.abspath(__file__)), "dist_device_dataset_worker.py")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29617", worker, str(tmp_path)]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    assert "world=2" in r.stdout and "bit-identical on every rank" in r.stdout, r.stdout[-500:]


@pytest.mark.gpu
def test_trainer_loop_with_the_device_dataset_runs_at_the_engine_rate(tmp_path):
    """At batch 512 the train_audio loop on a resident dataset stays within 1.3x of the same steps driven directly through
    Engine.train_step on batches already on the device."""
    import time
    import torch
    from tcresnet_b200 import train_audio
    make_split(tmp_path, "train", per_label=400)                              # 4,405 samples: 8 steps of 512 per epoch
    steps = 60
    args = _args(tmp_path, extra=f"--device_dataset --batch_size 512 --max_step_from_restore {steps}")
    trainer = train_audio.train(args)
    model = trainer.model
    fetch = {"step_op": trainer.train_op, "global_step": trainer.global_step, "total_loss": model.total_loss, "model_loss": model.model_loss}
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for _ in range(200):
        trainer.session.run(fetch)
    model.flush_feed()
    torch.cuda.synchronize()
    loop_ms = (time.perf_counter() - t0) / 200 * 1e3
    eng = model.engine
    wavs = [model.dataset.device_data.batch(i * 512, 0, 1234, 512)[0] for i in range(2)]
    hots = [model.dataset.device_data.batch(i * 512, 0, 1234, 512)[1] for i in range(2)]
    for i in range(20):
        eng.train_step(wavs[i % 2], hots[i % 2], model.params, model.slots, model.moving, 0.1, 0.9, 1e-3, dropout_seed=i)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for i in range(200):
        eng.train_step(wavs[i % 2], hots[i % 2], model.params, model.slots, model.moving, 0.1, 0.9, 1e-3, dropout_seed=i)
    torch.cuda.synchronize()
    direct_ms = (time.perf_counter() - t0) / 200 * 1e3
    print(f"train_audio loop on the resident dataset {loop_ms:.3f} ms/step, Engine.train_step directly {direct_ms:.3f} ms/step")
    assert loop_ms <= 1.3 * direct_ms
