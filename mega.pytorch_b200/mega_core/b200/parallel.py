"""Frame-parallel sharding of one video stream over `world` GPUs (SURVEY.md section 8e).

Key frame t of a group of `world` consecutive key frames is owned by rank t mod world: the owner runs the
per-frame branch of the (look-ahead local, global) frame pair that arrives with it; the fixed-size
payloads are exchanged with one all-gather whose output order IS the frame order, so every rank then
ingests the same frames in the same order and all replicas hold identical state (no reductions:
results are independent of `world`)."""
import torch
import torch.distributed as dist


def owner_of(key_frame, world):
    return key_frame % world


def frames_of_step(step, world):
    """key frames produced by distributed step `step` (in ingestion order)"""
    return list(range(step * world, (step + 1) * world))


# diagnostics: when COMM_EVENTS[0] is a list, every device all-gather appends its (start, end) CUDA events to it
# (bench.py's per-rank breakdown of a multi-GPU step; never set inside a timed region)
COMM_EVENTS = [None]


def gather_payloads(payload, out=None, group=None):
    """all-gather equal-size 1-D payloads -> [world, n] in rank (= frame) order. NCCL on GPUs
    (`all_gather_into_tensor`), gloo for the CPU tests of this host logic."""
    world = dist.get_world_size(group)
    if out is None:
        out = torch.empty(world, payload.numel(), dtype=payload.dtype, device=payload.device)
    if payload.is_cuda:
        rec = COMM_EVENTS[0]
        if rec is not None:
            a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            a.record()
        dist.all_gather_into_tensor(out.view(-1), payload.contiguous(), group=group)
        if rec is not None:
            b.record()
            rec.append((a, b))
    else:
        parts = [out[i] for i in range(world)]
        dist.all_gather(parts, payload.contiguous(), group=group)
    return out


# ----------------------------------------------------------------------------------------------------------------
# Wavefront schedule (SURVEY.md section 8e, option ii). The long-range memory couples the key frames of a group, but
# only as a depth-3 wavefront: what frame t pushes into stage s's memory depends on stage s-1's memory of frames < t
# (roi_box_feature_extractors.py:678-688, :913-928), never on its own stage. So the owner of frame t can run the
# whole aggregation of its frame alone if, before stage s reads its memory, it has applied the stage-s increments of
# the group's EARLIER frames (received by one small all-gather per stage) and only those: the ring slots that the
# group's LATER frames will overwrite must still hold the frames they are about to evict, exactly as in the
# sequential order "read, then push". After its last read a rank applies the remaining increments (its own included),
# which leaves every rank with the same ring as sequential processing of the whole group.
def wave_tables(mem_pushed, rank, world, rows0, rows12, mem_frames, base0, base12, baseb12):
    """Destination-row tables of one wavefront step, for the rank that owns frame `rank` of a group of `world` frames.

    mem_pushed : frames pushed into the memory before the group (identical on all ranks)
    rows0 / rows12 : rows per frame of the stage-0 memory (75) / of the stage-1 and stage-2 memories (15)
    mem_frames : ring capacity in frames (25); 0 without a long-range memory: the schedule has no increment stages, so
        the tables are empty and every frame sees no memory
    base0 / base12 / baseb12 : first ring row inside the stage-0 feature+box buffers, the stage-1/2 feature buffers and
        the stage-1/2 box buffers
    Returns int32 numpy arrays; entry [g * rows + j] is the destination row of row j of frame g's increment, or -1
    (= skipped by mega_copy_rows): `pre*` hold the frames g < rank, `post*` the frames g >= rank.
    `valid[g]` = memory frames frame g sees (the soft-max's key count is local rows + valid * rows)."""
    import numpy as np
    assert 0 <= rank < world and (mem_frames == 0 or world <= mem_frames), \
        "a group must fit the memory ring (its frames take distinct slots)"
    out = {}
    stages = (("0", rows0, base0), ("12", rows12, base12), ("b12", rows12, baseb12)) if mem_frames else ()
    for name, rows, base in stages:
        pre = np.full(world * rows, -1, dtype=np.int32)
        post = np.full(world * rows, -1, dtype=np.int32)
        for g in range(world):
            slot = (mem_pushed + g) % mem_frames
            dst = base + slot * rows + np.arange(rows, dtype=np.int32)
            (pre if g < rank else post)[g * rows:(g + 1) * rows] = dst
        out["pre" + name], out["post" + name] = pre, post
    out["valid"] = np.asarray([min(mem_pushed + g, mem_frames) for g in range(world)], dtype=np.int32)
    return out


def drive(gen, group=None):
    """run one rank's wavefront generator: every value it yields is (payload, gathered_out); the all-gather result is
    sent back in. Returns the generator's return value."""
    try:
        msg = next(gen)
        while True:
            payload, out = msg
            gather_payloads(payload.view(-1), out, group)
            msg = gen.send(out)
    except StopIteration as stop:
        return stop.value


def play(gens):
    """single-process stand-in for `drive` over all ranks of a group (tests: the ranks of an N-GPU group played on one
    device, or on the CPU for the host logic): advances the generators in lockstep and performs each all-gather by
    copying. Returns the list of return values in rank order."""
    world = len(gens)
    msgs, results, done = [None] * world, [None] * world, [False] * world
    for r, g in enumerate(gens):
        try:
            msgs[r] = next(g)
        except StopIteration as stop:
            results[r], done[r] = stop.value, True
    while not all(done):
        assert not any(done), "ranks left the wavefront at different collectives"
        parts = [m[0].reshape(-1).clone() for m in msgs]
        for r, g in enumerate(gens):
            out = msgs[r][1]
            for q in range(world):
                out[q].copy_(parts[q])
            try:
                msgs[r] = g.send(out)
            except StopIteration as stop:
                results[r], done[r] = stop.value, True
    return results


# ---------------------------------------------------------------------------------------------- wavefront self-check
# Before a multi-GPU run switches to the wavefront schedule, every rank can replay this check on its own device without
# any communication: random (but valid) window / global-pool state and frame payloads, the sequential owner-mode step as
# the truth, both ranks of a 2-rank wavefront group played in-process; it passes only if every predictor output, every
# detection and every memory ring is bit-identical. The engines run with CUDA graphs on, over enough groups that each
# wavefront segment is executed eagerly, captured and replayed. Cheap: no backbone work is involved.
def _rand_boxes(gen, n, im_w, im_h):
    x1 = torch.rand(n, generator=gen) * (im_w - 80)
    y1 = torch.rand(n, generator=gen) * (im_h - 80)
    return torch.stack([x1, y1, x1 + 10 + torch.rand(n, generator=gen) * 60, y1 + 10 + torch.rand(n, generator=gen) * 60], 1)


def _rand_rows(eng, shape, gen, dtype):
    """seeded feature rows in the engine's row format (the strict engine keeps them split-fp16: ops.split16_encode)"""
    x = torch.randn(shape, generator=gen) * 0.5
    if getattr(eng, "split16_att", False):
        from . import ops
        return ops.split16_encode(x)
    return x.to(dtype)


def random_state(eng, seed, im_w, im_h):
    """put a MegaEngine into the state of a video whose window and global pool are full (memory still empty)"""
    gen = torch.Generator().manual_seed(seed)
    eng.reset()
    for _ in range(eng.L):
        eng._claim_slot()
    eng.win_x.copy_(_rand_rows(eng, eng.win_x.shape, gen, eng.win_x.dtype))
    eng.win_boxes.copy_(_rand_boxes(gen, eng.win_boxes.shape[0], im_w, im_h))
    eng.win_cnt.fill_(eng.KP - 3)
    eng.glob_x.copy_(_rand_rows(eng, eng.glob_x.shape, gen, eng.glob_x.dtype))
    eng.glob_pushed = eng.GF


def random_payload(eng, seed, im_w, im_h):
    """what a rank's per-frame branch hands to the gather: x300 | boxes | count | x75, filled with seeded noise"""
    gen = torch.Generator().manual_seed(seed)
    p = torch.zeros_like(eng.payload_in)
    px, pb, pc, pg = eng._payload_views(p)
    px.copy_(_rand_rows(eng, px.shape, gen, px.dtype))
    pb.copy_(_rand_boxes(gen, pb.shape[0], im_w, im_h))
    pc.view(torch.int32)[0, 0] = eng.KP - 1 - seed % 4
    pg.copy_(_rand_rows(eng, pg.shape, gen, pg.dtype))
    return p


def wave_selfcheck(make_engine, im_w=1000, im_h=600, world=2, groups=3, seed=0, use_graph=True):
    """-> (ok, message). `make_engine()` must return fresh MegaEngines with identical weights on the current device."""
    def snap(eng, det):
        if eng.dev.type == "cuda":
            torch.cuda.synchronize(eng.dev)
        k, n = int(eng.cur_cnt.view(-1)[0]), int(det.count.reshape(-1)[0])
        return [eng.last_pred[:k].clone(), det.boxes[:n].clone(), det.scores[:n].clone(), det.labels[:n].clone()]

    solo = make_engine()
    ranks = [make_engine() for _ in range(world)]
    for e in [solo] + ranks:
        e.use_graph = use_graph
        random_state(e, seed, im_w, im_h)
    frames = groups * world
    payloads = [random_payload(solo, seed + 100 + t, im_w, im_h) for t in range(frames)]
    truth = [snap(solo, solo.dist_step(None, im_w, im_h, rank=0, world=1, payloads=payloads[t][None])[0])
             for t in range(frames)]
    if not any(t[1].shape[0] for t in truth):
        return False, "self-check is degenerate: the sequential step produced no detections"
    for t0 in range(0, frames, world):
        dets = play([ranks[r]._wave(None, im_w, im_h, r, world, payload=payloads[t0 + r]) for r in range(world)])
        for r in range(world):
            for i, (a, b) in enumerate(zip(truth[t0 + r], snap(ranks[r], dets[r]))):
                if not torch.equal(a, b):
                    return False, "key frame %d: %s differs from the sequential step" % (
                        t0 + r, ("predictor output", "boxes", "scores", "labels")[i])
    rings = {"E0": solo.KP + solo.nl0, "B0": solo.KP + solo.nl0, "Y1E": solo.nq, "Y2M": solo.nq, "B1": solo.nl12,
             "B2": solo.nl12, "win_x": 0, "win_boxes": 0, "win_cnt": 0, "glob_x": 0}
    for r in range(world):
        for name, off in rings.items():
            if not torch.equal(getattr(ranks[r], name)[off:], getattr(solo, name)[off:]):
                return False, "rank %d: ring %s differs from the sequential state" % (r, name)
    return True, "wavefront == sequential over %d key frames (bit-identical outputs and rings)" % frames
