import pytest

# A context may list one device several times: each entry has its own stream, workspaces, MSM lanes, twiddle tables and SRS
# shard, and the entries' work runs concurrently, so every multi-device path (sharded MSM, six-step NTT, row-range grand
# products and quotient passes, batch NTTs by polynomial) runs on one GPU. These are those aliased device lists.
ALIASED_DEVICE_LISTS = ([0, 0], [0, 0, 0], [0] * 8)


def device_lists(power_of_two=False):
    """pytest params of the device lists a multi-device test runs on: the aliased lists of device 0 always, and the real
    devices 0..min(count, 8) - 1, which skips where fewer than two GPUs are present. `power_of_two`: only the lists whose
    length is a power of two (a context of any other size takes the one-device NTT)."""
    import torch
    count = torch.cuda.device_count() if torch.cuda.is_available() else 0
    real = list(range(min(count, 8)))
    params = [pytest.param(ids, id="alias%d" % len(ids)) for ids in ALIASED_DEVICE_LISTS if not power_of_two or len(ids) & (len(ids) - 1) == 0]
    if power_of_two:
        real = real[:1 << (len(real).bit_length() - 1)] if real else real
    params.append(pytest.param(real, id="real", marks=pytest.mark.skipif(len(real) < 2, reason="needs >= 2 GPUs")))
    return params


@pytest.fixture(scope="session")
def be():
    """The product backend (CUDA). Fails loudly -- never falls back to the oracle."""
    import torch  # noqa: F401  (device presence check only)
    from spectre_b200 import halo2
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    b = halo2.Backend([0])
    yield b
    b.close()
