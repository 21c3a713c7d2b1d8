"""bin/rsem-run-em-batch and bin/rsem-run-gibbs-batch with RSEM_B200_DEVICES: every run with a list of lanes against the
same manifest run with the list unset.

A repeated device (0,0 and 0,0,0) runs several lanes on one card, so every case here runs on one GPU; 0,1 runs the same
comparisons where there are two.  rsem-run-gibbs-batch's files and standard output are byte for byte those of one lane (a
chain's draws depend only on its seed and its sample), and no two cooperative launches on one device overlap (the
lanes' RSEM_B200_TIMING stamps).  rsem-run-em-batch's files are compared at test_em_batch_exe_gpu's tolerances (the
counts of K12 and of the class-layout E-step are sums of atomic adds), each sample runs the same rounds, and the
blocks stay in manifest order.  The manifests mix both sides of each batch's size rule, and small arenas fill on every
lane."""
import filecmp
import os
import re
import shutil
import subprocess

import pytest

import rsem_files as rf
from test_dropin_gpu import CASES
from test_em_batch_arena_exe_gpu import _sample_bytes as _em_sample_bytes
from test_em_batch_exe_gpu import EXE as EM_EXE
from test_em_batch_exe_gpu import _blocks, _compare, _manifest
from test_gibbs_batch_arena_exe_gpu import _sample_bytes as _gibbs_sample_bytes
from test_gibbs_batch_exe_gpu import EXE as GIBBS_EXE
from test_gibbs_batch_exe_gpu import M, SPECS, _files, _threads

pytestmark = pytest.mark.gpu

# test_gibbs_batch_exe_gpu's samples and one above the batch's size rule (2^19 reads)
GIBBS_SPECS = SPECS + [(dict(N1=530000, N0=100), "1 3 1 -p 2 --seed 18 --pseudo-count 0.5")]


def _device_count():
    try:
        import rsem_b200
        return rsem_b200.load_library().device_count()
    except Exception:   # collected without a GPU or before the build
        return 0


def _lists(*lists):
    return [pytest.param(x, marks=pytest.mark.skipif(x == "0,1" and _device_count() < 2, reason="needs two GPUs"))
            for x in lists]


def _env(devices, arena=None, rounds=None):
    env = dict(os.environ, RSEM_B200_TIMING="1")
    for k in ("RSEM_B200_DEVICES", "RSEM_B200_DEVICE", "RSEM_B200_BATCH_ARENA_BYTES"):
        env.pop(k, None)
    if devices is not None:
        env["RSEM_B200_DEVICES"] = devices
    if arena is not None:
        env["RSEM_B200_BATCH_ARENA_BYTES"] = str(arena)
    if rounds is not None:
        env["RSEM_MAX_ROUND"], env["RSEM_MIN_ROUND"] = str(rounds), str(min(20, rounds))
    return env


def _lanes(stderr, tool):
    """(device, in the batch, on the single-sample path, arena full, [(start, end)] of the launches) per lane line"""
    out = []
    for m in re.finditer(rf"^{tool} timing: lane \d+, device (\d+): (\d+) samples in the batch, (\d+) on the single-sample "
                         r"path, arena full (\d+) times;.*?(?:launches(.*))?$", stderr, flags=re.M):
        stamps = [tuple(map(float, s.split("-"))) for s in (m.group(5) or "").split()]
        out.append((int(m.group(1)), int(m.group(2)), int(m.group(3)), int(m.group(4)), stamps))
    return out


def _totals(stderr, tool):
    m = re.search(rf"^{tool} timing: (\d+) samples in the batch, (\d+) on the single-sample path", stderr, flags=re.M)
    full = re.search(rf"^{tool} timing: arena full (\d+) times$", stderr, flags=re.M)
    assert m and full, stderr
    return int(m.group(1)), int(m.group(2)), int(full.group(1))


def _check_lanes(stderr, tool, devices):
    """one lane line per list entry (none for a list of one), adding up to the totals"""
    lanes = _lanes(stderr, tool)
    if devices is None or "," not in devices:
        assert lanes == [] and len(re.findall(rf"^{tool} timing:", stderr, flags=re.M)) == 3, stderr
        return lanes
    assert [x[0] for x in lanes] == [int(d) for d in devices.split(",")], stderr
    batched, single, full = _totals(stderr, tool)
    assert (sum(x[1] for x in lanes), sum(x[2] for x in lanes), sum(x[3] for x in lanes)) == (batched, single, full)
    return lanes


# ---- rsem-run-gibbs-batch ------------------------------------------------------------------------------------------------

@pytest.fixture(scope="module")
def gibbs_samples(built, tmp_path_factory):
    """GIBBS_SPECS after rsem-run-em-batch --gibbs-out, laid out as test_gibbs_batch_exe_gpu's samples"""
    root = tmp_path_factory.mktemp("lanes_gibbs")
    for k, (gen, _) in enumerate(GIBBS_SPECS):
        rf.gen_dataset(str(root / f"d{k}"), read_type=0, M=M, seed=7, sample_seed=200 + k, **gen)
    with open(root / "em_manifest", "w") as f:
        f.write("".join(f"d{k}/s d{k}/s.temp/s d{k}/s.stat/s --gibbs-out\n" for k in range(len(GIBBS_SPECS))))
    subprocess.run([EM_EXE, "d0/ref/r", "0", "em_manifest", "-q"], cwd=root, check=True, stdout=subprocess.DEVNULL,
                   env=_env(None))
    for k, (gen, _) in enumerate(GIBBS_SPECS):   # no alignable reads: the .ofg is the header, the model any sample's
        if gen["N1"] == 0:
            with open(root / f"d{k}" / "s.temp" / "s.ofg", "w") as f:
                f.write(f"{M} {gen['N0']}\n")
            shutil.copy(root / "d0" / "s.stat" / "s.model", root / f"d{k}" / "s.stat" / "s.model")
    with open(root / "prior.txt", "w") as f:
        f.write("".join(f"{0.05 + (i % 5) * 0.3:.2f} prior\n" for i in range(M)))
    return str(root)


def _gibbs_run(root, tag, ks, devices, arena=None):
    d = os.path.join(root, tag)
    shutil.copytree(os.path.join(root, "in"), d)
    with open(os.path.join(d, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {GIBBS_SPECS[k][1]}\n" for k in ks))
    p = subprocess.run([GIBBS_EXE, "d0/ref/r", "manifest"], cwd=d, env=_env(devices, arena), capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    return d, p


def _gibbs_same(a, b, ks):
    for k in ks:
        for f in _files(f"d{k}", _threads(GIBBS_SPECS[k][1])):
            assert filecmp.cmp(os.path.join(a, f"d{k}", f), os.path.join(b, f"d{k}", f), shallow=False), (k, f)


def _no_overlap(lanes):
    for dev in {x[0] for x in lanes}:
        spans = sorted(s for x in lanes if x[0] == dev for s in x[4])
        for (_, end), (start, _) in zip(spans, spans[1:]):
            assert start >= end, (dev, spans)


@pytest.mark.parametrize("arena", ["default", "one", "none"])
@pytest.mark.parametrize("devices", _lists("0", "0,0", "0,0,0", "0,1"))
def test_gibbs_lanes_match_one_device(gibbs_samples, tmp_path, devices, arena):
    """every manifest line.  "one": the arena of the largest batched sample, so some lane's arena fills (which lane
    takes which lines depends on timing, so no lane in particular is sure to fill).  "none": 1 byte, so every sample
    inside the size rule finds its lane's arena full, whichever lane takes it, and runs on the single-sample path"""
    root = str(tmp_path)
    shutil.copytree(gibbs_samples, root + "/in")
    ks = list(range(len(GIBBS_SPECS)))
    size = {"default": None, "none": 1}.get(arena)
    if arena == "one":
        size = max(b for b in _gibbs_sample_bytes(root + "/in") if b is not None)
    base, p0 = _gibbs_run(root, "base", ks, None, size)
    d, p = _gibbs_run(root, "lanes", ks, devices, size)
    assert p.stdout == p0.stdout
    _gibbs_same(d, base, ks)
    want = (0, 7) if arena == "none" else (4, 3)
    assert _totals(p.stderr, "rsem-run-gibbs-batch")[:2] == _totals(p0.stderr, "rsem-run-gibbs-batch")[:2] == want
    lanes = _check_lanes(p.stderr, "rsem-run-gibbs-batch", devices)
    if lanes:
        _no_overlap(lanes)
        assert sum(len(x[4]) for x in lanes) >= 4   # every single-sample run and at least one batch launch
    if arena == "one":
        assert _totals(p.stderr, "rsem-run-gibbs-batch")[2] >= 1
    if arena == "none":
        assert _totals(p.stderr, "rsem-run-gibbs-batch")[2] == 4


def test_gibbs_more_lanes_than_samples(gibbs_samples, tmp_path):
    root = str(tmp_path)
    shutil.copytree(gibbs_samples, root + "/in")
    ks = [0, 2]
    base, p0 = _gibbs_run(root, "base", ks, None)
    d, p = _gibbs_run(root, "lanes", ks, "0,0,0")
    assert p.stdout == p0.stdout
    _gibbs_same(d, base, ks)
    lanes = _check_lanes(p.stderr, "rsem-run-gibbs-batch", "0,0,0")   # every lane reports, idle or not
    assert sum(x[1] + x[2] for x in lanes) == 2
    _no_overlap(lanes)


# ---- rsem-run-em-batch ---------------------------------------------------------------------------------------------------

def _em_run(root, samples, tag, rt, devices, arena=None, rounds=None):
    d = os.path.join(root, tag)
    os.makedirs(d)
    for s, _ in samples:
        shutil.copytree(s, os.path.join(d, os.path.basename(s)))
    with open(os.path.join(d, "manifest"), "w") as f:
        for s, extra in samples:
            b = os.path.basename(s)
            f.write(" ".join([f"{b}/s", f"{b}/s.temp/s", f"{b}/s.stat/s", *extra]) + "\n")
    p = subprocess.run([EM_EXE, "s0/ref/r", str(rt), "manifest", "-p", "2"], cwd=d, env=_env(devices, arena, rounds),
                       capture_output=True, text=True)
    assert p.returncode == 0, p.stderr[-3000:]
    blocks = _blocks(p.stdout)
    assert [b[0].split()[2] for b in blocks] == [os.path.basename(s) + "/s" for s, _ in samples]   # manifest order
    return d, p, [sum(line.startswith("ROUND = ") for line in b) for b in blocks]


def _em_same(samples, a, b):
    for s, extra in samples:
        n = os.path.basename(s)
        _compare(os.path.join(a, n), os.path.join(b, n), "--gibbs-out" in extra, "-b" in extra)


@pytest.mark.parametrize("devices", _lists("0,0", "0,0,0", "0,1"))
@pytest.mark.parametrize("rounds", [13, 3, None])
@pytest.mark.parametrize("name", ["se_noq", "se_q_rspd_polyA", "pe_noq", "pe_q_rspd"])
def test_em_lanes_match_one_device(tmp_path, built, name, rounds, devices):
    """test_em_batch_exe_gpu's manifests; free-running se_noq adds a sample over K12's layout (the whole-GPU path)"""
    rt, opts = CASES[name]
    os.makedirs(tmp_path / "in")
    samples = _manifest(tmp_path / "in", rt, opts, wide=(name == "se_noq" and rounds is None))
    base, p0, rounds0 = _em_run(str(tmp_path), samples, "base", rt, None, rounds=rounds)
    d, p, rounds1 = _em_run(str(tmp_path), samples, "lanes", rt, devices, rounds=rounds)
    assert rounds1 == rounds0
    if rounds is not None:
        assert all(r in (0, rounds) for r in rounds1) and rounds1.count(rounds) == len(samples) - 1
    _em_same(samples, d, base)
    assert _totals(p.stderr, "rsem-run-em-batch")[:2] == _totals(p0.stderr, "rsem-run-em-batch")[:2]
    _check_lanes(p.stderr, "rsem-run-em-batch", devices)


@pytest.mark.parametrize("devices", _lists("0,0", "0,1"))
def test_em_lanes_small_arena(tmp_path, built, devices):
    """the arena of the second largest sample on every lane: the largest finishes on its lane's context, and some lane's
    arena fills (which lane takes which lines depends on timing)"""
    rt, opts = CASES["pe_q_rspd"]
    os.makedirs(tmp_path / "in")
    samples = _manifest(tmp_path / "in", rt, opts, wide=False)
    samples = samples + [(s + "_b", extra) for s, extra in samples[1:]]   # enough samples to fill two arenas
    for s, _ in samples[len(samples) - 4:]:
        shutil.copytree(s[:-2], s)
    one = sorted(b for b in _em_sample_bytes(samples, rt) if b is not None)[-2]
    base, p0, rounds0 = _em_run(str(tmp_path), samples, "base", rt, None, arena=one)
    d, p, rounds1 = _em_run(str(tmp_path), samples, "lanes", rt, devices, arena=one)
    assert rounds1 == rounds0
    _em_same(samples, d, base)
    batched, single, full = _totals(p.stderr, "rsem-run-em-batch")
    assert (batched, single) == _totals(p0.stderr, "rsem-run-em-batch")[:2] and single >= 1 and full >= 1
    _check_lanes(p.stderr, "rsem-run-em-batch", devices)


# ---- refusals ------------------------------------------------------------------------------------------------------------

def test_unopenable_device_writes_nothing(gibbs_samples, tmp_path):
    """RSEM_B200_DEVICES=0,99: exit status 255, a message naming device 99, no sample file of either tool"""
    shutil.copytree(gibbs_samples, tmp_path / "g")
    before = set(os.listdir(tmp_path / "g" / "d0" / "s.temp"))
    with open(tmp_path / "g" / "manifest", "w") as f:
        f.write(f"d0/s.temp/s d0/s.stat/s {GIBBS_SPECS[0][1]}\n")
    p = subprocess.run([GIBBS_EXE, "d0/ref/r", "manifest"], cwd=tmp_path / "g", env=_env("0,99"), capture_output=True,
                       text=True)
    assert p.returncode == 255 and "device 99" in p.stderr, p.stderr
    assert set(os.listdir(tmp_path / "g" / "d0" / "s.temp")) == before

    rt, opts = CASES["se_noq"]
    d = str(tmp_path / "e")
    rf.gen_dataset(d, read_type=rt, **dict(opts, seed=7))
    with open(os.path.join(d, "manifest"), "w") as f:
        f.write("s s.temp/s s.stat/s --gibbs-out\n")
    before = {x: set(os.listdir(os.path.join(d, x))) for x in ("s.temp", "s.stat")}
    p = subprocess.run([EM_EXE, "ref/r", str(rt), "manifest"], cwd=d, env=_env("0,99"), capture_output=True, text=True)
    assert p.returncode == 255 and "device 99" in p.stderr, p.stderr
    assert {x: set(os.listdir(os.path.join(d, x))) for x in ("s.temp", "s.stat")} == before


# ---- a lane that fails -----------------------------------------------------------------------------------------------------
# An output path taken by a directory makes one sample's writer fail on the host, after its K12 / K13 run: the run ends
# with status 255 and one message naming the device and the sample, and no sample block is printed.

def test_gibbs_lane_failure_names_device_and_sample(gibbs_samples, tmp_path):
    root = str(tmp_path)
    shutil.copytree(gibbs_samples, root + "/in")
    os.makedirs(os.path.join(root, "in", "d0", "s.temp", "s.countvectors0"))   # d0 runs in a batch: a writer thread fails
    d = os.path.join(root, "lanes")
    shutil.copytree(os.path.join(root, "in"), d)
    with open(os.path.join(d, "manifest"), "w") as f:
        f.write("".join(f"d{k}/s.temp/s d{k}/s.stat/s {GIBBS_SPECS[k][1]}\n" for k in range(len(SPECS))))
    p = subprocess.run([GIBBS_EXE, "d0/ref/r", "manifest"], cwd=d, env=_env("0,0"), capture_output=True, text=True,
                       timeout=600)
    assert p.returncode == 255, p.stderr[-3000:]
    assert p.stderr.strip().splitlines()[-1] == ("rsem-run-gibbs-batch: device 0, sample d0/s.temp/s (manifest line 1): "
                                                 "Cannot open d0/s.temp/s.countvectors0 for writing!"), p.stderr[-3000:]
    assert p.stdout == ""


def test_em_lane_failure_names_device_and_sample(tmp_path, built):
    rt, opts = CASES["se_noq"]
    os.makedirs(tmp_path / "in")
    samples = _manifest(tmp_path / "in", rt, opts, wide=False)
    os.makedirs(os.path.join(samples[3][0], "s.temp", "s.iso_res"))   # s3 finishes in a K12 batch, then its writer fails
    d = str(tmp_path / "lanes")
    os.makedirs(d)
    for s, _ in samples:
        shutil.copytree(s, os.path.join(d, os.path.basename(s)))
    with open(os.path.join(d, "manifest"), "w") as f:
        for s, extra in samples:
            b = os.path.basename(s)
            f.write(" ".join([f"{b}/s", f"{b}/s.temp/s", f"{b}/s.stat/s", *extra]) + "\n")
    p = subprocess.run([EM_EXE, "s0/ref/r", str(rt), "manifest", "-p", "2"], cwd=d, env=_env("0,0"), capture_output=True,
                       text=True, timeout=600)
    assert p.returncode == 255, p.stderr[-3000:]
    assert p.stderr.strip().splitlines()[-1] == ("rsem-run-em-batch: device 0, sample s3/s (manifest line 4): "
                                                 "Cannot open s3/s.temp/s.iso_res!"), p.stderr[-3000:]
    assert "== sample " not in p.stdout   # only the shared loaders' own lines, which they print as they run
