"""The NN-field likelihood kernels start while the kernel before them drains (programmatic dependent launch, engine.cu:
launch_pdl) and wait for it before their first global read.  Guards, eagerly and inside a captured CUDA graph:

* a torch kernel on the same stream writes the poses or the scan right before measure_device, and the records must be
  those of the written inputs.  The writing kernel is tiny and triggers its dependents only when it completes, so
  these cases check that the launch path keeps stream order; they are unlikely to catch a missing wait;
* two back-to-back calls must each return their own records.  With lik_kernel_nf_pm, two ~14 us grids share the
  per-particle accumulators (the fold leaves them at zero for the next call): this is the case a missing wait would
  break."""
import numpy as np
import pytest

from mcl_3dl_b200 import engine, synth

pytestmark = pytest.mark.gpu

P, N_LIK = 1024, 96  # >= 256 particles: lik_kernel_nf_pm; a scene of 64 particles runs lik_kernel_nf


def as_i32(a):
    b = np.ascontiguousarray(a).view(np.uint8).reshape(-1)
    assert b.size % 4 == 0
    return b.view(np.int32)


@pytest.fixture(scope="module")
def setup():
    torch = pytest.importorskip("torch")
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    s = synth.scene(50_000, P, N_LIK, 0, seed=11)
    other = synth.scene(50_000, P, N_LIK, 0, seed=12)
    eng = engine.Engine((0,))
    eng.set_map(s["map"], engine.LikParams(dist_weight=(1, 1, 5)), None)
    yield torch, eng, s, other
    eng.close()


def run(torch, eng, d_p, d_l, n_particles, d_out):
    dev = d_p.device
    d_b = torch.zeros(16, dtype=torch.uint8, device=dev)
    d_o = torch.zeros(6, dtype=torch.float32, device=dev)
    eng.measure_device(d_p.data_ptr(), n_particles, d_l.data_ptr(), N_LIK, d_b.data_ptr(), 0, d_o.data_ptr(), 2,
                       d_out.data_ptr(), torch.cuda.current_stream().cuda_stream)


def records(torch, d_out):
    torch.cuda.synchronize()
    return d_out.cpu().numpy().view(np.uint8).tobytes()


def reference(torch, eng, parts, lik, n_particles):
    d_p = torch.from_numpy(as_i32(parts)).cuda()
    d_l = torch.from_numpy(as_i32(lik)).cuda()
    d_out = torch.zeros(n_particles * 6, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    run(torch, eng, d_p, d_l, n_particles, d_out)
    return records(torch, d_out)


@pytest.mark.parametrize("n_particles", [P, 64])
@pytest.mark.parametrize("what", ["poses", "scan"])
@pytest.mark.parametrize("graph", [False, True])
def test_input_written_by_the_kernel_before(setup, n_particles, what, graph):
    torch, eng, s, other = setup
    parts, lik = s["particles"][:n_particles], s["lik"]
    want = reference(torch, eng, parts, lik, n_particles)
    # the other scene's inputs sit in the buffers until the torch kernel overwrites them
    src = torch.from_numpy(as_i32(parts if what == "poses" else lik)).cuda()
    stale_p = torch.from_numpy(as_i32(other["particles"][:n_particles])).cuda()
    stale_l = torch.from_numpy(as_i32(other["lik"])).cuda()
    d_p, d_l = stale_p.clone(), stale_l.clone()
    d_p = d_p if what == "poses" else torch.from_numpy(as_i32(parts)).cuda()
    d_l = d_l if what == "scan" else torch.from_numpy(as_i32(lik)).cuda()
    dst = d_p if what == "poses" else d_l
    stale = stale_p if what == "poses" else stale_l
    d_out = torch.zeros(n_particles * 6, dtype=torch.int32, device="cuda")

    def step():
        torch.add(src, 0, out=dst)  # an elementwise kernel, the last thing before measure_device on the stream
        run(torch, eng, d_p, d_l, n_particles, d_out)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for _ in range(2):
            dst.copy_(stale)
            d_out.zero_()
            torch.cuda.synchronize()
            g.replay()
            assert records(torch, d_out) == want
    else:
        for _ in range(2):
            dst.copy_(stale)
            d_out.zero_()
            torch.cuda.synchronize()
            step()
            assert records(torch, d_out) == want


@pytest.mark.parametrize("n_particles", [P, 64])
@pytest.mark.parametrize("graph", [False, True])
def test_back_to_back_calls_return_their_own_records(setup, n_particles, graph):
    torch, eng, s, other = setup
    scenes = [(s["particles"][:n_particles], s["lik"]), (other["particles"][:n_particles], other["lik"])]
    want = [reference(torch, eng, p, lk, n_particles) for p, lk in scenes]
    assert want[0] != want[1]
    dev_in = [(torch.from_numpy(as_i32(p)).cuda(), torch.from_numpy(as_i32(lk)).cuda()) for p, lk in scenes]
    outs = [torch.zeros(n_particles * 6, dtype=torch.int32, device="cuda") for _ in scenes]
    torch.cuda.synchronize()

    def step():
        for (d_p, d_l), d_out in zip(dev_in, outs):
            run(torch, eng, d_p, d_l, n_particles, d_out)
    if graph:
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g):
            step()
        for o in outs:
            o.zero_()
        g.replay()
    else:
        step()
    assert [records(torch, o) for o in outs] == want
