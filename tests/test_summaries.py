"""TensorBoard summaries of train_audio.py / evaluate_audio.py (common/tf_events.py, metrics/manager.py Summaries).

CPU: the event file's TFRecord framing and protos, read back by our reader and by TensorBoard's EventAccumulator; the tag table,
collections and firing steps against a restatement of the reference's schedule (helper/trainer.py:374-385), through the trainer's
own pending-summary logic with a model stub that reports losses `lag` steps late as the host-feed pipeline does.
GPU: train_audio / evaluate_audio runs whose event files hold the losses and metrics the runs logged and returned."""
import argparse
import logging
import os
import shlex
import struct
import subprocess
import sys
from collections import deque
from types import SimpleNamespace

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(HERE)
sys.path.insert(0, os.path.join(ROOT, "tc-resnet_b200"))
import tcresnet_b200  # noqa: E402,F401
from tcresnet_b200.common import tf_events as E  # noqa: E402
from tcresnet_b200.common.tf_bundle import crc32c, unmask_crc  # noqa: E402
from tcresnet_b200.helper.trainer import SingleLabelAudioTrainer  # noqa: E402
from tcresnet_b200.metrics import manager as M  # noqa: E402

ea = pytest.importorskip("tensorboard.backend.event_processing.event_accumulator")


def _files(d):
    return sorted(p for p in os.listdir(d) if p.startswith("events.out.tfevents."))


def _accumulator(path):
    acc = ea.EventAccumulator(str(path), size_guidance={ea.AUDIO: 0, ea.SCALARS: 0, ea.TENSORS: 0})
    acc.Reload()
    return acc


def _scalars(path):
    """{tag: {step: float32 value}} from our reader."""
    out = {}
    for ev in E.read_events(path):
        for tag, v in ev.get("summary", {}).items():
            if "simple_value" in v:
                out.setdefault(tag, {})[ev["step"]] = np.float32(v["simple_value"])
    return out


def _clips(n=6, frames=16000, seed=0):
    pcm = np.random.RandomState(seed).randint(-32768, 32768, (n, frames)).astype(np.int16)
    return pcm, (pcm / 32768.0).astype(np.float32)[..., None]          # decode_wav's scaling


# ------------------------------------------------------------------------------------------------ event file
def test_records_have_valid_masked_crcs_and_read_back(tmp_path):
    w = E.EventWriter(tmp_path)
    vals = np.float32([0.1, -3.75e-7, 1e30, np.pi])
    for step, v in enumerate(vals, 1):
        w.add(step, [E.scalar_value("a/b", v)])
    w.close()
    name = _files(tmp_path)
    assert len(name) == 1 and name[0].startswith("events.out.tfevents.") and w.path.name == name[0]
    data = w.path.read_bytes()
    pos, records = 0, 0
    while pos < len(data):                                   # the framing, checked here without the reader
        (n,) = struct.unpack("<Q", data[pos:pos + 8])
        assert unmask_crc(struct.unpack("<I", data[pos + 8:pos + 12])[0]) == crc32c(data[pos:pos + 8])
        assert unmask_crc(struct.unpack("<I", data[pos + 12 + n:pos + 16 + n])[0]) == crc32c(data[pos + 12:pos + 12 + n])
        pos, records = pos + 16 + n, records + 1
    assert pos == len(data) and records == 5
    evs = E.read_events(w.path)
    assert evs[0]["file_version"] == "brain.Event:2" and all("summary" in e for e in evs[1:])
    got = _scalars(w.path)["a/b"]
    assert {s: v.tobytes() for s, v in got.items()} == {s: v.tobytes() for s, v in enumerate(vals, 1)}     # bit-equal
    acc = _accumulator(w.path)
    assert acc.Tags()["scalars"] == ["a/b"]
    assert [(e.step, np.float32(e.value).tobytes()) for e in acc.Scalars("a/b")] == [(s, v.tobytes()) for s, v in enumerate(vals, 1)]
    bad = bytearray(data)
    bad[-6] ^= 1                                             # one bit of the last payload
    (tmp_path / "bad").write_bytes(bytes(bad))
    with pytest.raises(ValueError, match="payload CRC"):
        E.read_events(tmp_path / "bad")


@pytest.mark.parametrize("max_outputs", [1, 5])
def test_audio_summary_decodes_to_the_clips_samples(tmp_path, max_outputs):
    pcm, clips = _clips()
    w = E.EventWriter(tmp_path)
    w.add(7, E.audio_values("wav/train", clips, 16000, max_outputs))
    w.close()
    tags = [f"wav/train/audio/{i}" for i in range(max_outputs)] if max_outputs > 1 else ["wav/train/audio"]
    acc = _accumulator(w.path)
    assert sorted(acc.Tags()["audio"]) == sorted(tags)
    for i, tag in enumerate(tags):
        (a,) = acc.Audio(tag)
        assert a.step == 7 and a.content_type == "audio/wav" and a.sample_rate == 16000 and a.length_frames == 16000
        got, rate = E.decode_wav(a.encoded_audio_string)
        assert rate == 16000 and got.shape == (16000, 1) and np.array_equal(got[:, 0], pcm[i])
    ours = E.read_events(w.path)[1]["summary"]
    assert sorted(ours) == sorted(tags) and ours[tags[0]]["audio"]["num_channels"] == 1


def test_audio_encoding_rounds_and_clamps_like_tensorflow():
    got, _ = E.decode_wav(E.encode_wav(np.float32([[0.0], [0.5], [-1.0], [1.0], [2.0], [-2.0], [1.5 / 32768]]), 16000))
    assert got[:, 0].tolist() == [0, 16384, -32768, 32767, 32767, -32768, 2]


def test_config_text_lists_the_sorted_arguments(tmp_path):
    s = M.Summaries(tmp_path, 3)
    s.setup_experiment(argparse.Namespace(zeta=1, alpha=[1, 2], mid=None, beta="x"))
    s.close()
    want = [["alpha", "[1, 2]"], ["beta", "x"], ["mid", "None"], ["zeta", "1"]]
    (ours,) = [e for e in E.read_events(s.writer.path) if "summary" in e]
    assert ours["summary"]["config"]["plugin_name"] == "text" and ours["summary"]["config"]["tensor"].tolist() == want
    acc = _accumulator(s.writer.path)
    assert acc.Tags()["tensors"] == ["config"] and acc.SummaryMetadata("config").plugin_data.plugin_name == "text"
    from tensorboard.util import tensor_util
    assert tensor_util.make_ndarray(acc.Tensors("config")[0].tensor_proto).astype(str).tolist() == want


# ------------------------------------------------------------------------------------------------ tags and schedule
def _reference_collections(step, a):
    """helper/trainer.py:374-385, as written there."""
    keys = []
    if step >= a.step_min_summaries and step % a.step_save_summaries == 0:
        keys.append("SUMMARY_DEFAULT")
    if step % a.step_save_verbose_summaries == 0:
        keys.append("SUMMARY_VERBOSE")
    if step <= a.step_save_first_n_summaries:
        keys.append("SUMMARY_FIRST_N")
    return keys


def test_collections_follow_the_reference_schedule():
    a = SimpleNamespace(step_min_summaries=4, step_save_summaries=3, step_save_verbose_summaries=5, step_save_first_n_summaries=2)
    for step in range(0, 40):
        assert M.summary_collections(step, a.step_min_summaries, a.step_save_summaries, a.step_save_verbose_summaries,
                                     a.step_save_first_n_summaries) == _reference_collections(step, a)


def _table(is_training, learning_rate=True, exclude=()):
    m = M.AudioMetricManager(is_training, True, list(exclude))
    m.build_metric_ops({"dataset_split_name": "train", "label_names": ["a", "b"], "wavs": object(),
                        "losses": {"total_loss": 0, "model_loss": 0}, "learning_rate": object() if learning_rate else None})
    return m.summary_table


def test_tag_table_restates_the_reference_registration():
    d = "SUMMARY_DEFAULT"
    assert _table(True) == [("LossesMetricOp", "metric_loss/train/total_loss", "SCALAR", d),
                            ("LossesMetricOp", "metric_loss/train/model_loss", "SCALAR", d),
                            ("LearningRateSummaryOp", "learning_rate/train", "SCALAR", d),
                            ("WavSummaryOp", "wav/train", "AUDIO", d)]
    assert [r[1] for r in _table(False, learning_rate=False)] == ["metric_loss/train/total_loss", "metric_loss/train/model_loss"]
    assert [r[1] for r in _table(True, exclude=["WavSummaryOp"])] == ["metric_loss/train/total_loss",
                                                                      "metric_loss/train/model_loss", "learning_rate/train"]


class _StubModel:
    """What the trainer's summary path uses of the model: the step counter, the schedule, clips and losses reported `lag`
    steps after their step (the host-feed pipeline), and flush_feed."""

    def __init__(self, lag, clips):
        self.global_step, self.lag, self.clips = 0, lag, clips
        self.reported_losses, self._running, self._request, self._kept = deque(maxlen=256), [], 0, None
        self.lr_schedule = lambda step: 0.1 if step < 6 else 0.01

    def capture_clips(self, k):
        self._request = k

    def take_clips(self):
        kept, self._kept, self._request = self._kept, None, 0
        return kept

    @staticmethod
    def losses(step):
        return np.float32(1.0 / step), np.float32(2.0 / step)

    def step(self):
        self.global_step += 1
        if self._request:
            import torch
            self._kept = (torch.from_numpy(self.clips[self.global_step % 2][:self._request, :, 0].copy()), None)
            self._request = 0
        self._running.append(self.global_step)
        if len(self._running) > self.lag:
            s = self._running.pop(0)
            self.reported_losses.append((s, *self.losses(s)))

    def flush_feed(self):
        while self._running:
            s = self._running.pop(0)
            self.reported_losses.append((s, *self.losses(s)))


@pytest.mark.parametrize("max_outputs", [1, 5])
@pytest.mark.parametrize("lag,ckpt_step", [(0, 0), (2, 0), (2, 100)])
def test_trainer_writes_the_tag_table_at_the_firing_steps(tmp_path, max_outputs, lag, ckpt_step):
    """The trainer's own loop logic (prepare_step_summaries / write_step_summaries) on a stub model: each firing step's losses,
    learning rate and first max_outputs clips under their tags at that step, losses that arrive late included."""
    pcm = [_clips(6, 800, seed)[0] for seed in (1, 2)]
    model = _StubModel(lag, [(p / 32768.0).astype(np.float32)[..., None] for p in pcm])
    model.global_step = ckpt_step
    a = SimpleNamespace(step_min_summaries=4, step_save_summaries=3, step_save_verbose_summaries=5, step_save_first_n_summaries=2,
                        max_outputs=max_outputs)
    t = object.__new__(SingleLabelAudioTrainer)
    t.args, t.model, t.global_step_from_checkpoint, t._pending_summaries = a, model, ckpt_step, {}
    t.metric_manager = M.AudioMetricManager(True, False, [], summary=M.Summaries(tmp_path, max_outputs, 800))
    t.metric_manager.build_metric_ops({"dataset_split_name": "train", "label_names": ["a"], "wavs": object(),
                                       "losses": {"total_loss": 0, "model_loss": 0}, "learning_rate": object()})
    steps = 20
    for _ in range(steps):
        summary = t.prepare_step_summaries()
        model.step()
        if summary is not None:
            t._pending_summaries[summary[0]] = (summary[1], summary[2], model.take_clips())
        t.write_step_summaries()
    model.flush_feed()
    t.write_step_summaries(final=True)
    t.metric_manager.close_summaries()

    firing = [s for s in range(1, steps + 1) if "SUMMARY_DEFAULT" in _reference_collections(s, a)]
    assert firing == [6, 9, 12, 15, 18]                          # the short schedule: DEFAULT alone holds summaries
    (path,) = [tmp_path / f for f in _files(tmp_path)]
    got = _scalars(path)
    want_steps = [ckpt_step + s for s in firing]
    assert sorted(got) == ["learning_rate/train", "metric_loss/train/model_loss", "metric_loss/train/total_loss"]
    for g in want_steps:
        total, mloss = _StubModel.losses(g)
        assert got["metric_loss/train/total_loss"][g].tobytes() == total.tobytes()
        assert got["metric_loss/train/model_loss"][g].tobytes() == mloss.tobytes()
        assert got["learning_rate/train"][g] == np.float32(0.1 if g - 1 < 6 else 0.01)
    assert all(sorted(v) == want_steps for v in got.values())
    acc = _accumulator(path)
    tags = [f"wav/train/audio/{i}" for i in range(max_outputs)] if max_outputs > 1 else ["wav/train/audio"]
    assert sorted(acc.Tags()["audio"]) == sorted(tags)
    for i, tag in enumerate(tags):
        events = acc.Audio(tag)
        assert [e.step for e in events] == want_steps
        for e in events:
            assert np.array_equal(E.decode_wav(e.encoded_audio_string)[0][:, 0], pcm[e.step % 2][i])
    steps_written = [e["step"] for e in E.read_events(path)]
    assert steps_written == sorted(steps_written)              # in step order


def test_evaluation_summaries_hold_every_scalar_result(tmp_path):
    m = M.AudioMetricManager(False, True, [], summary=M.Summaries(tmp_path / "valid", 3))
    labels = ["a", "b", "c"]
    counts = np.zeros(11, np.int64)
    counts[[0, 4, 5, 8]] = [3, 2, 1, 4]
    counts[9], counts[10] = 5, 10
    m.evaluate_and_aggregate_metrics(1234, {"metric_counts": counts, "label_names": labels,
                                            "ranking": np.arange(10) / 10.0}, {"total_loss": np.float32([[0.5], [0.25]])})
    m.write_evaluation_summaries(1234)
    (path,) = [tmp_path / "valid" / f for f in _files(tmp_path / "valid")]    # flushed before close
    res = m.get_evaluation_result(1234)
    got = _scalars(path)
    want = {k: v for k, v in res.items() if np.isscalar(v)}
    assert set(got) == set(want) and "confusion_matrix" not in got
    assert {"accuracy", "top5_accuracy", "total_loss", "mAP/macro", "precision/a", "recall/b", "f1score/c", "ap/a"} <= set(got)
    for k, v in want.items():
        assert got[k] == {1234: np.float32(v)}, k
    m.close_summaries()


def test_summary_directories_follow_the_reference():
    assert M.summary_directory("/x/run", True, "valid").as_posix() == "/x/run"
    assert M.summary_directory(HERE, False, "valid").as_posix() == f"{HERE}/valid"
    assert M.summary_directory(f"{HERE}/test_summaries.py", False, "valid").as_posix() == f"{HERE}/valid"


# ------------------------------------------------------------------------------------------------ GPU: the CLIs end to end
COMMON = ("--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 40 --clip_duration_ms 1000 "
          "--window_size_ms 40 --window_stride_ms 20 ")


class _Records(logging.Handler):
    def __init__(self):
        super().__init__()
        self.lines = []

    def emit(self, record):
        self.lines.append(record.getMessage())


def _logged_losses(lines):
    """{global step: (TotalLoss, ModelLoss)} from the trainer's step log lines (the losses of the step they name)."""
    out = {}
    for line in lines:
        if "TotalLoss" not in line:
            continue
        step = int(line.split("GlobalStep")[1].split("/")[0])
        if "(losses of step" in line:
            step = int(line.split("(losses of step")[1].split(")")[0])
        if step > 0:                                            # before the first losses arrive the line shows step 0's NaNs
            out[step] = (float(line.split("TotalLoss")[1].split("/")[0]), float(line.split("ModelLoss")[1].split("|")[0]))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("device_dataset", [False, True])
def test_train_and_evaluate_tcresnet_leave_the_logged_values(tmp_path, device_dataset):
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio, train_audio
    make_split(tmp_path, "train", per_label=6, seed=0)
    make_split(tmp_path, "valid", per_label=3, seed=1)
    run = tmp_path / "run"
    dd = "--device_dataset " if device_dataset else ""
    args = train_audio.parse_arguments(shlex.split(
        f"--dataset_path {tmp_path} --dataset_split_name train {COMMON} --train_dir {run} --num_silent 8 "
        "--augmentation_method anchored_slice_or_pad_with_shift --batch_size 16 --boundaries 7 --max_step_from_restore 12 "
        "--lr_list 0.1 0.01 --absolute_schedule --no-boundaries_epoch --step_save_checkpoint 100 --step_evaluation 6 "
        "--step_save_summaries 1 --step_save_first_n_summaries 0 --max_outputs 2 --evaluation_iterations 2 "
        f"--optimizer mom --momentum 0.9 {dd}TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    from tcresnet_b200.common.utils import get_logger
    rec = _Records()
    get_logger("AudioTrainer").addHandler(rec)                   # the trainer's logger, set up as the trainer sets it up
    try:
        trainer = train_audio.train(args)
    finally:
        logging.getLogger("AudioTrainer").removeHandler(rec)
    trainer.model.engine.close()
    (path,) = [run / f for f in _files(run)]
    got = _scalars(path)
    logged = _logged_losses(rec.lines)
    assert len(logged) >= 8
    for step, (total, model_loss) in logged.items():           # the losses of every step, as the log line printed them
        assert round(float(got["metric_loss/train/total_loss"][step]), 5) == pytest.approx(total, abs=1.5e-5), step
        assert round(float(got["metric_loss/train/model_loss"][step]), 5) == pytest.approx(model_loss, abs=1.5e-5), step
    assert sorted(got["metric_loss/train/total_loss"]) == list(range(1, 13))
    assert {s: float(v) for s, v in got["learning_rate/train"].items()} == {s: float(np.float32(0.1 if s - 1 <= 7 else 0.01))
                                                                           for s in range(1, 13)}
    for step in (6, 12):                                        # the in-training evaluations
        res = trainer.metric_manager.results[step]
        for k, v in res.items():
            if np.isscalar(v):
                assert got[k][step] == np.float32(v), (k, step)
    acc = _accumulator(path)
    assert sorted(acc.Tags()["audio"]) == ["wav/train/audio/0", "wav/train/audio/1"]
    clips = acc.Audio("wav/train/audio/0")
    assert [e.step for e in clips] == list(range(1, 13))
    assert all(len(E.decode_wav(e.encoded_audio_string)[0]) == 16000 for e in clips)
    assert any(np.abs(E.decode_wav(e.encoded_audio_string)[0]).max() > 0 for e in clips)
    assert acc.Tags()["tensors"] == ["config"]

    latest = sorted(run.glob("*.index"))[-1].with_suffix("")
    eargs = evaluate_audio.parse_arguments(shlex.split(
        f"--dataset_path {tmp_path} --dataset_split_name valid {COMMON} --checkpoint_path {latest} --num_silent 6 "
        "--augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 --batch_size 3 "
        f"--no-shuffle --valid_type once --no-save_best_keeper {dd}TCResNet8Model --weight_decay 0.001 --width_multiplier 1.0"))
    (res,) = evaluate_audio.main(eargs)
    (epath,) = [run / "valid" / f for f in _files(run / "valid")]
    got = _scalars(epath)
    want = {k: v for k, v in res.items() if np.isscalar(v)}
    assert set(got) == set(want) and {"accuracy", "top5_accuracy", "mAP/macro", "mAP/samples", "total_loss"} <= set(got)
    for k, v in want.items():
        assert got[k] == {12: np.float32(v)}, k


@pytest.mark.gpu
def test_evaluate_dscnn_checkpoint_leaves_its_metrics(tmp_path):
    from oracle import dscnn_oracle as D
    from test_device_dataset import make_split
    from tcresnet_b200 import evaluate_audio
    from tcresnet_b200.common import checkpoint as ckpt
    make_split(tmp_path, "valid", per_label=3, seed=2)
    spec = D.build_spec("S", 49, 10, 12)
    values = D.init_variables(spec, 11)
    path = ckpt.save(tmp_path / "run", "DSCNNSModel", 1000, {k: v.astype(np.float32) for k, v in values.items()}, fmt="tf")
    args = evaluate_audio.parse_arguments(shlex.split(
        "--output_name output/softmax --num_classes 12 --preprocess_method mfcc --num_mfccs 10 --clip_duration_ms 1000 "
        f"--window_size_ms 40 --window_stride_ms 20 --dataset_path {tmp_path} --dataset_split_name valid --checkpoint_path {path} "
        "--num_silent 6 --augmentation_method anchored_slice_or_pad --background_frequency 0.0 --background_max_volume 0.0 "
        "--batch_size 3 --no-shuffle --valid_type once --no-save_best_keeper DSCNNSModel"))
    (res,) = evaluate_audio.main(args)
    (epath,) = [tmp_path / "run" / "valid" / f for f in _files(tmp_path / "run" / "valid")]
    got = _scalars(epath)
    want = {k: v for k, v in res.items() if np.isscalar(v)}
    assert set(got) == set(want) and "accuracy" in got
    for k, v in want.items():
        assert got[k] == {1000: np.float32(v)}, k
    config = [e for e in E.read_events(epath) if "config" in e.get("summary", {})]
    assert len(config) == 1 and ["model", "DSCNNSModel"] in config[0]["summary"]["config"]["tensor"].tolist()


@pytest.mark.gpu
def test_data_parallel_training_writes_one_event_file(tmp_path):
    """Two ranks under torchrun: rank 0 writes the summaries, the other rank opens no writer."""
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs >= 2 GPUs")
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29617", os.path.join(ROOT, "tc-resnet_b200", "train_audio.py"),
           "--dataset_path", "synthetic:1024", "--dataset_split_name", "train", "--train_dir", str(tmp_path),
           "--augmentation_method", "anchored_slice_or_pad_with_shift", "--batch_size", "64", "--boundaries", "1000",
           "--max_step_from_restore", "6", "--lr_list", "0.1", "0.01", "--absolute_schedule", "--no-boundaries_epoch",
           "--step_save_checkpoint", "100", "--step_evaluation", "3", "--step_save_summaries", "1", "--optimizer", "mom",
           "--momentum", "0.9", "--data_parallel"] + shlex.split(COMMON) + ["TCResNet8Model", "--weight_decay", "0.001"]
    r = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-4000:]
    (path,) = [tmp_path / f for f in _files(tmp_path)]
    got = _scalars(path)
    assert sorted(got["metric_loss/train/total_loss"]) == list(range(1, 7)) and 3 in got["accuracy"] and 6 in got["accuracy"]
