"""rsem-run-em-batch and rsem-run-gibbs-batch with RSEM_B200_DEVICES on the CPU: a bad manifest line is refused before any
device of the list is opened, so the refusal names the line, not the device that cannot be opened."""
import os
import subprocess

import rsem_files as rf


def _env():
    env = dict(os.environ, RSEM_B200_DEVICES="0,99")
    env.pop("RSEM_B200_DEVICE", None)
    return env


def test_em_batch_manifest_refused_before_devices(built, tmp_path):
    rf.gen_dataset(str(tmp_path / "d0"), read_type=0, M=60, N1=300, N0=10, sample_seed=1)
    with open(tmp_path / "manifest", "w") as f:
        f.write("d0/s d0/s.temp/s d0/s.stat/s\nd1/s d1/s.temp/s\n")
    p = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-em-batch"), "d0/ref/r", "0", "manifest"], cwd=tmp_path, env=_env(),
                       capture_output=True, text=True)
    assert p.returncode == 255 and "manifest line 2:" in p.stderr and "device" not in p.stderr, p.stderr
    assert not os.path.exists(tmp_path / "d0" / "s.stat" / "s.theta")


def test_gibbs_batch_manifest_refused_before_devices(built, tmp_path):
    rf.gen_dataset(str(tmp_path / "d0"), read_type=0, M=60, N1=300, N0=10, sample_seed=1)
    with open(tmp_path / "manifest", "w") as f:
        f.write("d0/s.temp/s d0/s.stat/s 2 4 0\n")   # GAP must be at least 1
    p = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch"), "d0/ref/r", "manifest"], cwd=tmp_path, env=_env(),
                       capture_output=True, text=True)
    assert p.returncode == 255 and "manifest line 1: GAP must be at least 1!" in p.stderr and "device" not in p.stderr, p.stderr
    assert not os.path.exists(tmp_path / "d0" / "s.temp" / "s.countvectors0")
