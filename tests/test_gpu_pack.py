"""The two writers of the centre pack agree.  bkm_finalize_step builds the next iteration's pack of the device-resident
Lloyd loop; bkm_pack_centers builds the pack every other call reads.  For the same centres both must write the same
bytes, on both size paths (one kernel for small k*d; the globals, then the layouts for large k*d) and for every set of
layouts a shape carries (float64; fp32 with and without the family-1 operands; bf16 with the family-3 operands)."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu

# (dtype of the rows, k, d)
SHAPES = [("float32", 256, 64), ("float32", 100, 41), ("float32", 20, 13), ("float32", 512, 64), ("float32", 4096, 32),
          ("float64", 20, 13), ("float64", 3000, 32),
          ("bfloat16", 256, 64), ("bfloat16", 1024, 128), ("bfloat16", 4096, 128)]
FILL = 0xA5         # both packs start from this byte, so bytes that neither writer touches compare equal too


@pytest.fixture(scope="module")
def be():
    from dask_ml_b200.engine import CudaBackend

    return CudaBackend()


def _centres(be, k, d, seed):
    import torch

    rng = np.random.RandomState(seed)
    C = rng.standard_normal((k, d)) * rng.uniform(0.5, 20.0, size=(k, 1)) + rng.uniform(-50.0, 50.0, size=(1, d))
    return torch.from_numpy(C).to(be.device).contiguous()


def _filled_pack(be, C, dt):
    import torch

    nbytes = be.pack_centers(C, dt).numel()
    return torch.full((nbytes,), FILL, dtype=torch.uint8, device=be.device)


def _reduced(C):
    """[k*d sums | k counts | inertia] whose centre update is C itself: every count is 1."""
    import torch

    k = C.shape[0]
    return torch.cat([C.reshape(-1), torch.ones(k, dtype=torch.float64, device=C.device),
                      torch.zeros(1, dtype=torch.float64, device=C.device)])


def _bits(t):
    import torch

    return t.contiguous().view(torch.int64)


@pytest.mark.parametrize("dtype,k,d", SHAPES)
def test_finalize_step_pack_matches_pack_centers(be, dtype, k, d):
    import torch

    dt = getattr(torch, dtype)
    C = _centres(be, k, d, 1000 + k + d)
    c_in = _centres(be, k, d, 2000 + k + d)
    c_out = torch.full((k, d), float("nan"), dtype=torch.float64, device=be.device)
    want = _filled_pack(be, C, dt)
    be.pack_centers(C, dt, out=want)
    got = _filled_pack(be, C, dt)
    state, _ = be.loop_state_new(-1.0, 4)               # tol < 0: the update is always taken over
    be.finalize_step(_reduced(C), c_in, c_out, state, got, dt)
    torch.cuda.synchronize()
    done, n_iter, shift = be.loop_state_read(state)
    assert (done, n_iter) == (0, 1)
    assert shift == pytest.approx(float(((c_in - C) ** 2).sum()), rel=1e-12)
    assert torch.equal(_bits(c_out), _bits(C))
    diff = (got != want).nonzero()
    assert diff.numel() == 0, "pack bytes differ from byte %d on (%d bytes differ)" % (int(diff[0]), diff.numel())


@pytest.mark.parametrize("dtype,k,d", SHAPES)
def test_finalize_step_converged_keeps_pack(be, dtype, k, d):
    import torch

    dt = getattr(torch, dtype)
    C = _centres(be, k, d, 3000 + k + d)
    c_in = _centres(be, k, d, 4000 + k + d)
    c_out = torch.empty((k, d), dtype=torch.float64, device=be.device)
    want = _filled_pack(be, c_in, dt)
    be.pack_centers(c_in, dt, out=want)
    got = _filled_pack(be, c_in, dt)
    be.pack_centers(c_in, dt, out=got)
    state, _ = be.loop_state_new(float("inf"), 4)       # tol = inf: the first iteration converges
    for _ in range(2):                                  # the second call comes after convergence: a no-op
        be.finalize_step(_reduced(C), c_in, c_out, state, got, dt)
    torch.cuda.synchronize()
    done, n_iter, _ = be.loop_state_read(state)
    assert done != 0 and n_iter == 1
    assert torch.equal(got, want)
