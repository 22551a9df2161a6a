"""Per-world-size transport thresholds (mpi4jax_b200/_src/tuning.py): table lookup, file overrides,
crossover detection of the autotuner.  The reference has no counterpart (it calls MPI)."""

import json

import pytest

from mpi4jax_b200._src import tuning

H100 = "NVIDIA H100 80GB HBM3"


def test_default_table_covers_every_world_size():
    for world in (2, 3, 4, 6, 8, 16):
        t = tuning.thresholds(world, H100)
        assert set(t) == set(tuning.KEYS)
        assert t["ll_max"] <= 64 << 10            # the LL buffers hold 2 x 64 KiB per peer
    # the table compiled into the module is what the native library starts with: a communicator created
    # without a tuning file makes no extra native call
    assert tuning.thresholds(8, H100) == tuning.NATIVE_DEFAULTS
    # world sizes in between use the next smaller entry of the table
    assert tuning.thresholds(6, H100) == tuning.thresholds(4, H100)
    # an unknown GPU model falls back to the H100 numbers
    assert tuning.thresholds(8, "Some Other GPU") == tuning.thresholds(8, H100)


def test_tuning_file_overrides_entry_by_entry(tmp_path, monkeypatch):
    path = tmp_path / "box.json"
    path.write_text(json.dumps({"gpu": H100, "table": {"4": {"nvls_min": 1 << 20}, "8": {"ll_max": 32 << 10}}}))
    monkeypatch.setenv("MPI4JAX_B200_TUNING_FILE", str(path))
    base4 = dict(tuning._entry_for(tuning.DEFAULTS_BY_GPU[H100], 4))
    got4 = tuning.thresholds(4, H100)
    assert got4["nvls_min"] == 1 << 20 and got4["ll_max"] == base4["ll_max"]
    assert tuning.thresholds(8, H100)["ll_max"] == 32 << 10
    assert tuning.thresholds(2, H100)["nvls_min"] == 1 << 20     # 2 < 4: the file's smallest entry applies
    monkeypatch.setenv("MPI4JAX_B200_TUNING_FILE", str(tmp_path / "missing.json"))
    with pytest.raises(FileNotFoundError):
        tuning.thresholds(8)
    bad = tmp_path / "bad.json"
    bad.write_text(json.dumps({"table": {"8": {"warp_speed": 9}}}))
    monkeypatch.setenv("MPI4JAX_B200_TUNING_FILE", str(bad))
    with pytest.raises(ValueError, match="unknown tuning keys"):
        tuning.thresholds(8)


def test_crossover_detection():
    sizes = [1 << k for k in range(10, 20)]
    a = [5, 5, 6, 6, 8, 12, 20, 40, 80, 160]            # wins small
    b = [9, 9, 9, 9, 9, 10, 12, 16, 24, 40]
    assert tuning.crossover(sizes, a, b) == 1 << 14
    noisy_b = list(b)
    noisy_b[2] = 5.5                                     # one noisy sample does not end A's range
    assert tuning.crossover(sizes, a, noisy_b) == 1 << 14
    assert tuning.crossover(sizes, [x + 100 for x in a], b) == 0
    assert tuning.crossover(sizes, [1] * 10, b) == sizes[-1]
    assert tuning.crossover(sizes, [None] * 10, b) == 0
