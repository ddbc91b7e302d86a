"""2-GPU checks (pytest -m gpu on a box with >= 2 GPUs; skipped otherwise): the fused render + all-gather
(peer stores from the kernel epilogue into symmetric memory) equals per-rank renders gathered with NCCL."""
import os
import socket

import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

pytestmark = pytest.mark.gpu


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    torch.cuda.set_device(rank)
    dev = torch.device("cuda", rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=dev)
    try:
        import ml_gmpi_b200 as g
        from ml_gmpi_b200 import synth, dist as gdist
        flags = torch.zeros(1, dtype=torch.int32, device=dev)
        ok, maxdiff, mc_ok = True, 0.0, None
        # 3 views of 128^2 (30 tiles of 64x30: the direct kernel) and 4 views of 256^2 (144 tiles: the staged kernel)
        for B, N, R in ((4, 12, 256), (3, 12, 128)):
            case = synth.make_case(n_planes=N, tex=R, img=R, n_mpi=B, seed=100 + rank, device=dev)
            color, depth = g.render_views(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, color_minus1_1=True)
            ref = gdist.all_gather_frames(gdist.pack_frames(color, depth))          # NCCL path
            # NVLS multicast variant (one store per quad, the switch replicates), when the fabric has it
            try:
                fgm = gdist.FrameGather(B, R, R, dev, multicast=True)
            except RuntimeError:
                fgm = None
            if fgm is not None:
                fgm.render(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, flags, color_minus1_1=True)
                fgm.finish()
                torch.cuda.synchronize(dev)
                mc_ok = bool(torch.equal(fgm.frames, ref)) and mc_ok is not False
            fg = gdist.FrameGather(B, R, R, dev, multicast=False)
            for _ in range(2):                                                      # twice: buffers are reused
                fg.render(case.rgba, case.dhw, case.view2mpi, case.ray_dir, case.eye, case.z_dir, flags, color_minus1_1=True)
                fg.finish()
            torch.cuda.synchronize(dev)
            ok = ok and bool(torch.equal(fg.frames, ref))
            maxdiff = max(maxdiff, float((fg.frames - ref).abs().max()))
        # write-after-read across iterations (ADVICE r1): DIFFERENT data every step, ranks deliberately skewed, and a reader
        # of step k's frames still in flight on the render stream while the peers already run step k+1
        cases = [case, synth.make_case(n_planes=N, tex=R, img=R, n_mpi=B, seed=500 + rank, device=dev)]
        refs = []
        for c in cases:
            cc, dd = g.render_views(c.rgba, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, color_minus1_1=True)
            refs.append(gdist.all_gather_frames(gdist.pack_frames(cc, dd)))
        snaps = []
        for k in range(8):
            c = cases[k % 2]
            if (k + rank) % 2:
                torch.cuda._sleep(20_000_000)                                        # ~10 ms of skew on alternating ranks
            fg.render(c.rgba, c.dhw, c.view2mpi, c.ray_dir, c.eye, c.z_dir, flags, color_minus1_1=True)
            fg.finish()
            snap = fg.frames.clone()                                                 # the in-flight reader
            for _ in range(4):
                snap = snap + 0.0
            snaps.append(snap)
        torch.cuda.synchronize(dev)
        for k, snap in enumerate(snaps):
            if not torch.equal(snap, refs[k % 2]):
                ok = False
                maxdiff = max(maxdiff, float((snap - refs[k % 2]).abs().max()))
        q.put((rank, ok and mc_ok is not False, maxdiff, int(flags.item()), mc_ok))
    finally:
        dist.destroy_process_group()


def test_fused_gather_equals_nccl_all_gather():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    procs = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    for p in procs:
        p.start()
    res = [q.get(timeout=300) for _ in procs]
    for p in procs:
        p.join(timeout=120)
        assert p.exitcode == 0
    for rank, equal, maxdiff, fl, mc_ok in res:
        assert equal and fl == 0, (rank, equal, maxdiff, fl, mc_ok)
    print("multicast (NVLS) variant:", {r[0]: r[4] for r in res})
