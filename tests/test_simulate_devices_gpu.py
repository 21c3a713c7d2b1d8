"""bin/rsem-simulate-reads over several devices (RSEM_B200_DEVICES with more than one entry): the read files, the
.sim.*.results tables and stdout (with the resimulation count) must be byte-identical to the reference simulator's for
the same seed, i.e. to the stored digests of tests/golden/reference/sim_*.tar.xz that test_simulate_gpu.py checks one
device against.  Each device owns every G-th stream window and jumps its mt19937 state between them, so a wrong jump,
a wrong window split or a wrong hand-off of the entry point between devices changes the reads.

"0,0" and "0,0,0" run several contexts on one card and need one H100; "0,1" and "0,1,2" are skipped without the
GPUs.  Three devices do not divide the window count.  The cases: all four model types at theta0 0 and 0.2 (3000 reads,
all inside the first window: the other devices' windows are dropped), windows of 2500-5000 words (every device runs
many windows and hand-offs), failed attempts, the exact-body path (a reachable all-zero table row), 1 M reads at the
default window, and two seeds."""
import hashlib
import json
import os
import random
import shutil
import subprocess
import tarfile

import pytest

import rsem_files as rf

pytestmark = pytest.mark.gpu

BIN = os.path.join(rf.ROOT, "bin", "rsem-simulate-reads")
SETS = ["se_noq", "se_q_polyA", "pe_noq", "pe_q_rspd", "se_q_rspd"]  # model types 0, 1, 2, 3, 1 (estRSPD)
LISTS = ["0,0", "0,0,0", "0,1", "0,1,2"]


def _device_count():
    import rsem_b200
    return rsem_b200.load_library().device_count()


@pytest.fixture(params=LISTS)
def devices(request, built):
    need = max(int(d) for d in request.param.split(",")) + 1
    if _device_count() < need:
        pytest.skip(f"needs {need} GPUs")
    return request.param


# ---- the inputs test_simulate_gpu.py generates for each stored case (the stored digest of the inputs pins them) ----
def _golden(tmp_path, name):
    g = tmp_path / ("golden_" + name)
    if not g.exists():
        g.mkdir()
        with tarfile.open(os.path.join(rf.ROOT, "tests", "golden", name + ".tar.gz")) as t:
            t.extractall(g, filter="data")
    return g / name


def _results(path, M):
    rng = random.Random(7)
    lines = ["transcript_id\tgene_id\tlength\teffective_length\texpected_count\tTPM\tFPKM\tIsoPct"]
    for i in range(1, M + 1):
        tpm = 0.0 if i % 7 == 0 else rng.uniform(0, 100)
        lines.append(f"T{i}\tG\t1\t1\t1\t{tpm:.2f}\t0\t0")
    open(path, "w").write("\n".join(lines) + "\n")


def _case(tmp_path, key, name, model_lines=None):
    src = _golden(tmp_path, name)
    d = tmp_path / key
    shutil.copytree(src / "ref", d / "ref")
    lines = open(src / "out" / "model20").read().split("\n")
    open(d / "model", "w").write("\n".join(model_lines(lines) if model_lines else lines))
    M = int(open(d / "ref" / "r.ti").readline().split()[0])
    _results(d / "res.tsv", M)
    return d


def _zero_rspd_bins(lines):
    k = next(i for i in range(len(lines) - 2) if lines[i].strip() == "1" and lines[i + 1].strip() == "20"
             and len(lines[i + 2].split()) == 20)
    pdf = lines[k + 2].split()
    lines[k + 2] = " ".join(["0"] * 14 + pdf[14:])
    return lines


def _zero_profile_rows(lines):
    k = next(i for i, l in enumerate(lines) if l.strip() == "100" and len(lines[i + 1].split()) == 100)
    init = [float(x) for x in lines[k + 1].split()]
    q = max(range(100), key=lambda i: init[i])
    k0 = next(i for i, l in enumerate(lines) if l.strip() == "100 5")
    for r in range(5):
        lines[k0 + 1 + q * 6 + r] = " ".join(["0"] * 5)
    return lines


def _stored(key, d):
    """the reference's stdout and output digests for case `key`, after checking that d holds its inputs"""
    with tarfile.open(os.path.join(rf.REF_RUNS, key + ".tar.xz")) as tar:
        read = lambda n: tar.extractfile(n).read().decode()
        inputs, stdout, digests = read("inputs.sha256"), read("stdout"), json.loads(read("digests.json"))
    assert inputs == hashlib.sha256(repr(sorted(rf._tree_digests(str(d)).items())).encode()).hexdigest(), \
        f"{key}: the generated inputs differ from those the reference was run on"
    return stdout, digests


def _compare(d, key, theta0, n, seed, devices, window=None):
    stdout, digests = _stored(key, d)
    out = str(d) + ".gpu"
    shutil.rmtree(out, ignore_errors=True)
    os.makedirs(out)
    env = {**os.environ, "RSEM_B200_DEVICES": devices}
    env.pop("RSEM_B200_SIM_WINDOW", None)
    if window:
        env["RSEM_B200_SIM_WINDOW"] = str(window)
    p = subprocess.run([BIN, str(d / "ref" / "r"), str(d / "model"), str(d / "res.tsv"), str(theta0), str(n),
                        os.path.join(out, "s"), "--seed", str(seed)], capture_output=True, text=True, env=env)
    assert p.returncode == 0, p.stderr
    assert {f: hashlib.sha256(open(os.path.join(out, f), "rb").read()).hexdigest()
            for f in sorted(os.listdir(out))} == digests
    assert p.stdout == stdout
    return p


@pytest.mark.parametrize("name", SETS)
@pytest.mark.parametrize("theta0", [0.0, 0.2])
def test_model_types(tmp_path, devices, name, theta0):
    """3000 reads end inside the first window"""
    key = f"sim_{name}_{theta0}"
    _compare(_case(tmp_path, key, name), key, theta0, 3000, 11, devices)


@pytest.mark.parametrize("name", ["pe_q_rspd", "se_noq"])
def test_many_windows(tmp_path, devices, name):
    key = f"sim_win_{name}"
    _compare(_case(tmp_path, key, name), key, 0.1, 20000, 5, devices, window=3000)


def test_failed_attempts_many_windows(tmp_path, devices):
    key = "sim_rspd_fail_win"
    p = _compare(_case(tmp_path, key, "pe_q_rspd", _zero_rspd_bins), key, 0.1, 20000, 13, devices, window=2500)
    assert "Total number of resimulation is 0" not in p.stdout


def test_exact_body_many_windows(tmp_path, devices):
    key = "sim_zero_rows_win"
    _compare(_case(tmp_path, key, "pe_q_rspd", _zero_profile_rows), key, 0.2, 20000, 4, devices, window=5000)


def test_million_reads(tmp_path, devices):
    """windows of the default 2^22 words, far more than the devices"""
    p = _compare(_case(tmp_path, "sim_1m", "se_noq"), "sim_1m", 0.05, 1000000, 3, devices)
    assert "GEN 1000000" in p.stdout


def test_million_reads_timing_lines(tmp_path, built):
    """RSEM_B200_TIMING=1 prints each device's phases; the devices take turns, window by window"""
    d = _case(tmp_path, "sim_1m", "se_noq")
    out = str(d) + ".gpu"
    os.makedirs(out)
    env = {**os.environ, "RSEM_B200_DEVICES": "0,0", "RSEM_B200_TIMING": "1"}
    env.pop("RSEM_B200_SIM_WINDOW", None)
    p = subprocess.run([BIN, str(d / "ref" / "r"), str(d / "model"), str(d / "res.tsv"), "0.05", "1000000",
                        os.path.join(out, "s"), "--seed", "3", "-q"], capture_output=True, text=True, env=env)
    assert p.returncode == 0, p.stderr
    lines = [l for l in p.stderr.splitlines() if l.startswith("rsem-simulate-reads timing: device")]
    assert len(lines) == 2 and all("windows" in l for l in lines)
    windows = [int(l.rsplit(" ", 1)[1]) for l in lines]
    assert windows[0] >= 2 and windows[0] - windows[1] in (0, 1)
    assert "mt19937 jumps" in p.stderr


@pytest.mark.parametrize("seed", [1, 2])
def test_seeds(tmp_path, devices, seed):
    key = f"sim_seed{seed}"
    _compare(_case(tmp_path, key, "pe_noq"), key, 0.2, 2000, seed, devices)


def test_invalid_device_id(tmp_path, built):
    """a device that does not exist ends the run with status 255 and a message naming it"""
    d = _case(tmp_path, "sim_seed1", "pe_noq")
    env = {**os.environ, "RSEM_B200_DEVICES": "0,99"}
    p = subprocess.run([BIN, str(d / "ref" / "r"), str(d / "model"), str(d / "res.tsv"), "0.2", "2000",
                        str(tmp_path / "out"), "--seed", "1"], capture_output=True, text=True, env=env)
    assert p.returncode == 255, p.stderr
    assert "device 99" in p.stderr
