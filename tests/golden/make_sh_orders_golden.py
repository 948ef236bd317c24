"""Record tests/golden/sh_orders_golden.npz and soundspaces_b200/data/sh_hrtf_bank_order3.txt by running the reference's
closed-source ``scripts/AmbisonicBinauralizer`` (needs an upstream checkout in ``SOUNDSPACES_REFERENCE``):

* the 16 x 2 x 256 filter bank = the tool's responses (lags 128..383) to a unit impulse in each channel of a
  16-channel file at a block-aligned position, azimuth 0 (the route make_sh_golden.py takes for the 9-row bank);
* its outputs on seeded RIR-shaped (decaying) signals at K = 1, 4 and 16 channels and five azimuths;
* its outputs on block-aligned impulses in the third-order channels 9..15 at 37.5 and 90 degrees;
* a small seeded tree in scripts/ambisonic_to_binaural.py's layout (``<scene>/irs/*.wav``) converted by the tool at
  0, 90, 180 and 270 degrees: the output samples and the raw 44-byte output headers.  The tree holds one file per
  channel count, a PCM16 file, a 44.1 kHz file, one long enough for the FFT form, a WAVE_FORMAT_EXTENSIBLE file
  (which the tool refuses) and a file that is not a wav.
"""
import os
import struct
import subprocess
import sys
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, ROOT)
from oracle import sh_elf  # noqa: E402
from oracle.sh_orders import SH_DELAY, SH_TAPS  # noqa: E402

ORDERS_K = (1, 4, 16)
AZIMUTHS = (0.0, 90.0, 180.0, 270.0, 37.5)
N = 3072
IMPULSE_AZ = (37.5, 90.0)
IMPULSE_POS = 384
ANGLES = (0, 90, 180, 270)
# scene -> [(file name, channels, length, sample rate, kind, seed)]; kind: f32, pcm16, extensible or text
TREE = {
    "sceneA": [("0_1.wav", 1, 1200, 16000, "f32", 31), ("1_4.wav", 4, 2000, 16000, "f32", 32),
               ("2_4.wav", 4, 1000, 16000, "pcm16", 33), ("3_9.wav", 9, 1500, 16000, "extensible", 34),
               ("notes.txt", 0, 0, 0, "text", 0)],
    "sceneB": [("0_9.wav", 9, 1300, 44100, "f32", 35), ("1_16.wav", 16, 7500, 16000, "f32", 36)],
}


def make_amb(seed, K, n=N):
    """RIR-shaped: decaying noise (the tool's block convolver deviates more on full-length white signals)."""
    rng = np.random.default_rng(seed)
    env = np.exp(-np.arange(n) / (n / 5.0))[:, None]
    return (rng.standard_normal((n, K)) * env * 0.3).astype(np.float32)


def seed_of(K, az):
    return 100 * K + int(round(az * 10)) % 1000


def impulse(K, channel, n=1024):
    x = np.zeros((n, K), np.float32)
    x[IMPULSE_POS, channel] = 1.0
    return x


def tree_signal(K, n, kind, seed):
    x = make_amb(seed, K, n)
    if kind == "pcm16":
        return np.round(x * 20000.0).astype("<i2")
    return x


def write_wav(path, data, sr, kind):
    """f32: plain 16-byte fmt chunk, tag 3; pcm16: tag 1; extensible: tag 0xFFFE with a 40-byte fmt chunk."""
    data = np.ascontiguousarray(data)
    n, ch = data.shape
    payload = data.tobytes()
    bits = 8 * data.dtype.itemsize
    if kind == "extensible":
        ext = struct.pack("<HHI", 22, bits, 0) + bytes.fromhex("0300000000001000800000aa00389b71")   # float subformat
        fmt = struct.pack("<HHIIHH", 0xFFFE, ch, sr, sr * ch * bits // 8, ch * bits // 8, bits) + ext
    else:
        fmt = struct.pack("<HHIIHH", 1 if kind == "pcm16" else 3, ch, sr, sr * ch * bits // 8, ch * bits // 8, bits)
    with open(path, "wb") as f:
        f.write(b"RIFF" + struct.pack("<I", 4 + 8 + len(fmt) + 8 + len(payload)) + b"WAVE")
        f.write(b"fmt " + struct.pack("<I", len(fmt)) + fmt)
        f.write(b"data" + struct.pack("<I", len(payload)) + payload)


def write_tree(ambisonic_dir):
    """The seeded input tree, ``<ambisonic_dir>/<scene>/irs/<file>``.  Returns {(scene, name): input array}."""
    inputs = {}
    for scene, files in TREE.items():
        d = os.path.join(ambisonic_dir, scene, "irs")
        os.makedirs(d, exist_ok=True)
        for name, K, n, sr, kind, seed in files:
            if kind == "text":
                with open(os.path.join(d, name), "w") as f:
                    f.write("not an impulse response\n")
                continue
            x = tree_signal(K, n, kind, seed)
            write_wav(os.path.join(d, name), x, sr, kind)
            inputs[(scene, name)] = x
    return inputs


def main():
    p = 256
    bank = np.zeros((16, 2, SH_TAPS), dtype=np.float32)
    for k in range(16):
        imp = np.zeros((1024, 16), np.float32)
        imp[p, k] = 1.0
        y = sh_elf.binauralize(imp, 0.0)
        bank[k] = y[p + SH_DELAY: p + SH_DELAY + SH_TAPS].T
        assert not y[: p + SH_DELAY].any()
    out = {"bank": bank}
    for K in ORDERS_K:
        for az in AZIMUTHS:
            out[f"K{K}/az{az:g}"] = sh_elf.binauralize(make_amb(seed_of(K, az), K), az)
    for az in IMPULSE_AZ:
        for k in range(9, 16):
            out[f"imp/k{k}/az{az:g}"] = sh_elf.binauralize(impulse(16, k), az)
    with tempfile.TemporaryDirectory() as d:
        amb_dir, bin_dir = os.path.join(d, "ambisonic"), os.path.join(d, "binaural")
        write_tree(amb_dir)
        for scene in TREE:
            for angle in ANGLES:
                dst = os.path.join(bin_dir, scene, str(angle))
                subprocess.run([sh_elf.ELF, "-i", os.path.join(amb_dir, scene, "irs"), "-o", dst, "-a", str(angle)],
                               check=True, capture_output=True)
                names = sorted(os.listdir(dst))
                out[f"tree/{scene}/{angle}/files"] = np.array(names)
                for name in names:
                    with open(os.path.join(dst, name), "rb") as f:
                        raw = f.read()
                    out[f"tree/{scene}/{angle}/{name}/header"] = np.frombuffer(raw[:44], np.uint8)
                    out[f"tree/{scene}/{angle}/{name}/out"] = np.frombuffer(raw[44:], "<f4").reshape(-1, 2)
    np.savez_compressed(os.path.join(ROOT, "tests", "golden", "sh_orders_golden.npz"), **out)
    # rows 0-8 are the packaged second-order bank bit for bit; the product ships rows 9-15 as text
    assert np.array_equal(bank[:9], np.load(os.path.join(ROOT, "soundspaces_b200", "data", "sh_hrtf_bank.npy")))
    np.savetxt(os.path.join(ROOT, "soundspaces_b200", "data", "sh_hrtf_bank_order3.txt"), bank[9:].reshape(14, 256),
               fmt="%.9e", header="AmbisonicBinauralizer HRTF bank, rows 9-15 (third order, ACN) x 2 ears x 256 taps; "
                                  "one line per (row, ear)")
    print("bank energy per channel", (bank[:, 0].astype(np.float64) ** 2).sum(axis=1).round(3))


if __name__ == "__main__":
    main()
