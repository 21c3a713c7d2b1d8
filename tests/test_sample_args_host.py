"""rsem-run-gibbs and rsem-run-gibbs-batch refuse a sample by the same rule with the same message: the batch prefixes it with
"<manifest> line N: ", rsem-run-gibbs ends with it after the progress lines of what it loaded first.  All of these are
refused before a CUDA context is used, so this machine needs no GPU for them."""
import os
import subprocess

import pytest

import rsem_files as rf

M = 60
LOADED = "Refs.loadRefs finished!\nLoading data is finished!\nLoading group information is finished!\n"

# case: (manifest fields after the sample's imdName / statName, rsem-run-gibbs's stdout before the refusal)
CASES = {
    "nsamples": ("d1/s.temp/s d1/s.stat/s 4 1 1", ""),
    "gap": ("d1/s.temp/s d1/s.stat/s 4 6 0", ""),
    "no_omit": ("d2/s.temp/noomit d2/s.stat/s 4 6 1", LOADED),
    "bad_omit": ("d2/s.temp/badomit d2/s.stat/s 4 6 1", LOADED),
    "no_prior": ("d1/s.temp/s d1/s.stat/s 4 6 1 --prior missing_prior.txt", LOADED),
    "short_prior": ("d1/s.temp/s d1/s.stat/s 4 6 1 --prior short_prior.txt", LOADED),
}


@pytest.fixture(scope="module")
def root(built, tmp_path_factory):
    """three samples of one reference with the files rsem-run-gibbs reads (.ofg, .omit, .model), and broken variants"""
    root = tmp_path_factory.mktemp("gargs")
    for k in range(3):
        d = rf.gen_dataset(str(root / f"d{k}"), read_type=0, M=M, N1=50, N0=10, sample_seed=k + 1)
        with open(os.path.join(d, "s.temp", "s.ofg"), "w") as f:
            f.write(f"{M} 10\n" + "".join(f"0 0.5 {1 + i % M} 0.5\n" for i in range(50)))
        os.makedirs(os.path.join(d, "s.stat"), exist_ok=True)
        with open(os.path.join(d, "s.stat", "s.model"), "w") as f:
            f.write("0\n0.5\n")
    t = root / "d2" / "s.temp"
    for name in ("noomit", "badomit"):
        (t / f"{name}.ofg").write_text(f"{M} 0\n")
    (t / "badomit.omit").write_text(f"3 {M + 1}\n")
    (root / "short_prior.txt").write_text("".join("1.0\n" for _ in range(M - 1)))
    return str(root)


@pytest.mark.parametrize("case", list(CASES))
def test_one_rule_both_tools(root, case):
    fields, loaded = CASES[case]
    with open(os.path.join(root, "manifest"), "w") as f:
        f.write("d0/s.temp/s d0/s.stat/s 4 6 1 -p 2 --seed 3\n\n" + fields + "\n")
    env = dict(os.environ)
    env.pop("RSEM_B200_DEVICES", None)
    batch = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs-batch"), "d0/ref/r", "manifest"], cwd=root, env=env,
                           capture_output=True, text=True)
    assert batch.returncode == 255, batch.stderr
    assert batch.stderr.startswith("manifest line 3: "), batch.stderr
    why = batch.stderr[len("manifest line 3: "):]
    single = subprocess.run([os.path.join(rf.BIN_DIR, "rsem-run-gibbs"), "d0/ref/r", *fields.split()], cwd=root, env=env,
                            capture_output=True, text=True)
    assert single.returncode == 255, single.stderr
    assert single.stderr == why
    assert single.stdout == loaded
