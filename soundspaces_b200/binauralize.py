"""Ambisonic -> binaural RIR trees on the GPU: a drop-in for the reference's ``scripts/ambisonic_to_binaural.py``
(which runs the closed ``AmbisonicBinauralizer`` once per scene and angle, 160 subprocesses at a time).

``binauralize_tree`` converts every ``<scene>/irs/*.wav`` of an ambisonic tree into ``<scene>/<angle>/<same name>``
of the binaural tree that ``AudioRenderService`` reads, with the tool's file formats:

* input: RIFF/WAVE with a plain ``fmt `` chunk, IEEE float32 (tag 3) or PCM16 (tag 1, decoded as ``x / 32767`` like
  the tool, not librosa's ``/ 32768``), 1, 4, 9 or 16 channels (ambisonic orders 0 to 3, ACN).  Anything else, e.g.
  WAVE_FORMAT_EXTENSIBLE, gets a warning and no output, and the conversion goes on (the tool exits 0 on those too);
  files whose name does not end in ``.wav`` are ignored;
* output: float32 stereo with a plain 44-byte header, the input's sample-rate field and the input's length.

Files are grouped by (channel count, length bucket) and decoded in batches, every file at all its angles in one
call (``BatchedAudioRenderer.sh_decode_angles``).  Zero-padding a file to its bucket's length is exact: the decode is
causal and the output is cut at the input's length.  Reads and writes run on a thread pool; the decode of one batch
overlaps the host work of the next.

    python -m soundspaces_b200.binauralize [--ambisonic-dir data/ambisonic_rirs/mp3d]
        [--binaural-dir data/binaural_rirs/mp3d] [--angles 0 90 180 270] [--device cuda:0]
"""
from __future__ import annotations

import argparse
import os
import struct
import warnings
from collections import deque
from concurrent.futures import ThreadPoolExecutor

import numpy as np

SH_CHANNELS = (1, 4, 9, 16)
WAVE_FORMAT_PCM, WAVE_FORMAT_IEEE_FLOAT = 1, 3
PCM16_SCALE = 32767.0


class WavFormatError(ValueError):
    """A file the ambisonic converter does not read."""


def read_ambisonic_wav(path):
    """Returns (sample rate, (n, K) float32).  Raises :class:`WavFormatError` for a file the tool would not convert."""
    with open(path, "rb") as f:
        raw = f.read()
    if len(raw) < 12 or raw[:4] != b"RIFF" or raw[8:12] != b"WAVE":
        raise WavFormatError(f"{path}: not a RIFF/WAVE file")
    fmt = data = None
    pos = 12
    while pos + 8 <= len(raw) and (fmt is None or data is None):
        cid, size = raw[pos:pos + 4], struct.unpack_from("<I", raw, pos + 4)[0]
        body = raw[pos + 8:pos + 8 + size]
        if cid == b"fmt ":
            fmt = body
        elif cid == b"data":
            data = body
        pos += 8 + size + (size & 1)
    if fmt is None or len(fmt) < 16 or data is None:
        raise WavFormatError(f"{path}: no fmt or data chunk")
    tag, ch, sr, _, block_align, bits = struct.unpack_from("<HHIIHH", fmt)
    if (tag, bits) == (WAVE_FORMAT_IEEE_FLOAT, 32):
        dtype, scale = "<f4", None
    elif (tag, bits) == (WAVE_FORMAT_PCM, 16):
        dtype, scale = "<i2", PCM16_SCALE
    else:
        raise WavFormatError(f"{path}: format tag {tag} with {bits} bits (float32 or PCM16 only)")
    if ch not in SH_CHANNELS:
        raise WavFormatError(f"{path}: {ch} channels (1, 4, 9 or 16)")
    if block_align != ch * bits // 8:
        raise WavFormatError(f"{path}: block align {block_align} for {ch} x {bits} bits")
    n = len(data) // block_align
    x = np.frombuffer(data, dtype=dtype, count=n * ch).reshape(n, ch)
    x = x.astype(np.float32) / np.float32(scale) if scale else x.astype(np.float32)
    return sr, x


def wav_header(n, sr):
    """The tool's output header: RIFF, a 16-byte ``fmt `` chunk (tag 3, 2 channels, block align 8, 32 bits), data."""
    nbytes = n * 8
    return (b"RIFF" + struct.pack("<I", 36 + nbytes) + b"WAVE"
            + b"fmt " + struct.pack("<IHHIIHH", 16, WAVE_FORMAT_IEEE_FLOAT, 2, sr, sr * 8, 8, 32)
            + b"data" + struct.pack("<I", nbytes))


def write_binaural_wav(path, sr, data):
    """data: (n, 2) float32 -> the tool's float32 stereo wav."""
    data = np.ascontiguousarray(data, dtype="<f4")
    if data.ndim != 2 or data.shape[1] != 2:
        raise ValueError(f"binaural data must be (n, 2), got {data.shape}")
    with open(path, "wb") as f:
        f.write(wav_header(data.shape[0], sr))
        f.write(data.tobytes())


def angle_dir_name(angle):
    """``str(angle)`` of the script's integer angles; 37.5 -> ``37.5``."""
    return f"{float(angle):g}"


def angle_dir_done(irs_dir, angle_dir):
    """The script's skip rule: an angle directory is done when it holds as many entries as the input directory."""
    return os.path.isdir(angle_dir) and len(os.listdir(irs_dir)) == len(os.listdir(angle_dir))


def length_bucket(n):
    """Padded length of a batch holding an n-sample file: n rounded up to 1/8 of its power of two (>= 1024)."""
    q = max(1024, 1 << max(0, n.bit_length() - 4))
    return -(-n // q) * q


def binauralize_tree(ambisonic_dir, binaural_dir, angles=(0, 90, 180, 270), device="cuda:0",
                     max_batch_bytes=256 << 20, workers=8):
    """Convert ``<ambisonic_dir>/<scene>/irs/*.wav`` into ``<binaural_dir>/<scene>/<angle>/*.wav`` on ``device``.

    Like the script, an angle directory whose entry count already equals that of ``irs/`` is skipped, so a scene
    whose ``irs/`` also holds a file that produces no output is converted again on every run.  ``max_batch_bytes``
    bounds one batch's device input plus output.  Returns counts: ``converted`` input files, ``written`` output
    files, ``refused`` input files and ``skipped_dirs`` angle directories."""
    import torch

    from .renderer import BatchedAudioRenderer

    angles = [float(a) for a in angles]
    if not angles:
        raise ValueError("at least one angle")
    counts = {"converted": 0, "written": 0, "refused": 0, "skipped_dirs": 0}
    jobs = []                                  # (input path, [output paths], angle indices)
    for scene in sorted(os.listdir(ambisonic_dir)):
        irs = os.path.join(ambisonic_dir, scene, "irs")
        if not os.path.isdir(irs):
            continue
        todo = []
        for ai, a in enumerate(angles):
            d = os.path.join(binaural_dir, scene, angle_dir_name(a))
            if angle_dir_done(irs, d):
                counts["skipped_dirs"] += 1
            else:
                os.makedirs(d, exist_ok=True)
                todo.append(ai)
        if not todo:
            continue
        for name in sorted(os.listdir(irs)):
            if name.endswith(".wav") and os.path.isfile(os.path.join(irs, name)):
                outs = [os.path.join(binaural_dir, scene, angle_dir_name(angles[ai]), name) for ai in todo]
                jobs.append((os.path.join(irs, name), outs, tuple(todo)))
    if not jobs:
        return counts

    renderer = BatchedAudioRenderer(16000, 4096, device=device)
    dev = renderer.device
    az_sets = {}

    def read(job):
        try:
            return job, read_ambisonic_wav(job[0])
        except (OSError, ValueError, struct.error) as e:
            return job, e

    def write(files, host, done):
        done.synchronize()
        for i, (job, sr, n) in enumerate(files):
            for a, path in enumerate(job[1]):
                write_binaural_wav(path, sr, host[i, a, :n].numpy())

    def decode(key, files):
        K, Lb, todo = key
        n = len(files)
        stage = torch.zeros((n, Lb, K), dtype=torch.float32).pin_memory()
        for i, (_, x) in enumerate(files):
            stage[i, : x.shape[0]] = torch.from_numpy(x)
        if todo not in az_sets:
            az_sets[todo] = torch.tensor([angles[ai] for ai in todo], dtype=torch.float32)
        with torch.cuda.device(dev):
            out = renderer.sh_decode_angles(stage.to(dev, non_blocking=True), az_sets[todo])
            host = torch.empty(out.shape, dtype=torch.float32).pin_memory()
            host.copy_(out, non_blocking=True)
            done = torch.cuda.Event()
            done.record()
        return host, done

    pending = {}                               # (K, bucket, angle set) -> [(job, sr, samples)]
    writes = []
    with ThreadPoolExecutor(max_workers=workers) as pool:
        def flush(key):
            files = pending.pop(key)
            host, done = decode(key, [(job, x) for job, _, x in files])
            writes.append(pool.submit(write, [(job, sr, x.shape[0]) for job, sr, x in files], host, done))
            counts["converted"] += len(files)
            counts["written"] += sum(len(job[1]) for job, _, _ in files)

        reads = deque()
        for i in range(len(jobs)):
            while len(reads) < 4 * workers and i + len(reads) < len(jobs):      # bounded read-ahead
                reads.append(pool.submit(read, jobs[i + len(reads)]))
            job, res = reads.popleft().result()
            if isinstance(res, Exception):
                warnings.warn(f"not converted: {res}")
                counts["refused"] += 1
                continue
            sr, x = res
            key = (x.shape[1], length_bucket(x.shape[0]), job[2])
            group = pending.setdefault(key, [])
            group.append((job, sr, x))
            per_file = key[1] * (key[0] + 2 * len(key[2])) * 4
            if (len(group) + 1) * per_file > max_batch_bytes or (len(group) + 1) * len(key[2]) > 65535:
                flush(key)
            for w in [w for w in writes if w.done()]:
                w.result()                     # a failed write raises here
                writes.remove(w)
        for key in list(pending):
            flush(key)
        for w in writes:
            w.result()
    return counts


def main(argv=None):
    p = argparse.ArgumentParser(description="Convert an ambisonic RIR tree to binaural RIRs on the GPU "
                                            "(scripts/ambisonic_to_binaural.py on the AmbisonicBinauralizer).")
    p.add_argument("--ambisonic-dir", default=os.path.join("data", "ambisonic_rirs", "mp3d"))
    p.add_argument("--binaural-dir", default=os.path.join("data", "binaural_rirs", "mp3d"))
    p.add_argument("--angles", type=float, nargs="+", default=[0, 90, 180, 270])
    p.add_argument("--device", default="cuda:0")
    args = p.parse_args(argv)
    counts = binauralize_tree(args.ambisonic_dir, args.binaural_dir, args.angles, args.device)
    print(" ".join(f"{k}={v}" for k, v in counts.items()))


if __name__ == "__main__":
    main()
