"""Wavefront multi-GPU step of the MEGA engine (SURVEY.md section 8e, option ii), as a mixin of MegaEngine.

Rank r aggregates ONLY its own key frame of a group of `world` frames. The memory increments of the group (75 + 15 + 15
rows per frame) travel in one small all-gather per relation stage; before stage s reads its memory the rank applies the
increments of the group's earlier frames, after its last read the rest (the reference's "read, then push" order). This
replaces the replicated "state" part of dist_step (~0.7 ms per foreign frame) by three latency-bound collectives. The
launches of the rank's own frame are those of MegaEngine._aggregate_split(owner), so detections are bit-identical to
dist_step for any world size. Schedule tables, the NCCL / in-process drivers and the self-check live in parallel.py; the
evidence (symbolic proof, engine code on CPU stand-ins, gloo, bit-identity on one GPU) is listed in DESIGN.md section 6."""
import torch

from . import ops


def _with_precision(fn):
    import functools

    @functools.wraps(fn)
    def wrapper(self, *a, **k):
        with ops.precision(self.cfg.precision):
            return fn(self, *a, **k)
    return wrapper


class WavefrontMixin:
    def _wave_alloc(self, world):
        if getattr(self, "_wave_world", None) == world:
            return
        R, A = self.R, self.A
        z = lambda *s, dtype=torch.float32: torch.zeros(*s, device=self.dev, dtype=dtype)
        self.w_ld = self.fw + 4                              # 32-bit words per increment row: feature row | box
        self.w_inc = [z(R, self.w_ld), z(A, self.w_ld), z(A, self.w_ld)]
        self.w_all = [z(world, R * self.w_ld), z(world, A * self.w_ld), z(world, A * self.w_ld)]
        self._wtab_off, off = {}, 0
        for name, n in (("pre0", R), ("post0", R), ("pre12", A), ("post12", A), ("preb12", A), ("postb12", A)):
            self._wtab_off[name] = (off, world * n)
            off += world * n
        self._wtab_ring = [torch.zeros(off, dtype=torch.int32).pin_memory() for _ in range(4)]
        self._wtab_ev = [None] * 4
        self.wtab_d = z(off, dtype=torch.int32)
        self._wave_world, self._wave_steps = world, 0

    def _wtab(self, name):
        o, n = self._wtab_off[name]
        return self.wtab_d[o:o + n]

    def _wave_fill(self, rank, world):
        """destination-row tables of this group (host -> pinned ring -> device), from the memory counter at group start"""
        from . import parallel
        tabs = parallel.wave_tables(self.mem_pushed, rank, world, self.R, self.A, self.MEMF, self.KP + self.nl0, self.nq,
                                    self.nl12)
        ring = self._wave_steps % len(self._wtab_ring)
        if self._wtab_ev[ring] is not None:
            self._wtab_ev[ring].synchronize()
        host = self._wtab_ring[ring]
        for name, (o, n) in self._wtab_off.items():
            host[o:o + n].copy_(torch.from_numpy(tabs[name]))
        self.wtab_d.copy_(host, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        self._wtab_ev[ring] = ev
        self._wave_steps += 1

    def _inc_views(self, buf):
        """[rows, fw + 4] words -> (feature rows [rows, D] in the activation dtype, boxes [rows, 4])"""
        w = buf.view(-1, self.w_ld)
        x = w[:, :self.feat_dim] if self.act == torch.float32 else w.view(self.act)[:, :self.feat_dim]
        return x, w[:, self.fw:]

    def _wave_pack(self, stage, x_rows, box_rows):
        x, b = self._inc_views(self.w_inc[stage])
        n = x.shape[0]
        with ops.copy_batch():
            ops.copy_rows(x_rows, x, n)
            ops.copy_rows(box_rows, b, n)

    def _wave_apply(self, stage, which, x_dst, box_dst):
        """scatter the gathered increments of the group into the memory rings; `which`: "pre" / "post" """
        x, b = self._inc_views(self.w_all[stage])
        n = x.shape[0]
        with ops.copy_batch():
            ops.copy_rows(x, x_dst, n, dst_idx=self._wtab(which + ("0" if stage == 0 else "12")))
            ops.copy_rows(b, box_dst, n, dst_idx=self._wtab(which + ("0" if stage == 0 else "b12")))

    @_with_precision
    def _wave_ingest(self, payload):
        """one frame of the group enters the window / global pool (no aggregation)"""
        self.payload_in.copy_(payload, non_blocking=True)
        slot_new = self._claim_slot()
        gslot = self.glob_pushed % self.GF
        self.glob_pushed += 1
        self._fill_tables(slot_new=slot_new, gslot=gslot)
        self._graph_run(("wave_ingest",), self._payload_to_rings)

    @_with_precision
    def _wave_seg(self, seg, key, im_w, im_h):
        return self._graph_run(("wave", seg) + key, lambda: getattr(self, "_wave_" + seg)(im_w, im_h))

    def _wave_a(self, im_w, im_h):
        """window of the own key frame, global stage G0, stage-0 increment (needs no memory)"""
        KP, R, nl0 = self.KP, self.R, self.nl0
        E0 = self.E0
        self._assemble_window()
        self._attention(self.att_g[0], E0[KP:KP + nl0], nl0, self.glob_x, self.GF * R, self.ld_g, E0[KP:KP + nl0])
        self._attention(self.att_g[0], E0[:KP], KP, self.glob_x, self.GF * R, self.ld_g, E0[:KP], reuse_kv=True)
        ops.gather_rows(E0, self.idx_qin0, self.Qin0, self.nq)
        self._wave_pack(0, E0[KP:KP + R], self.B0[KP:KP + R])

    def _wave_b(self, im_w, im_h):
        """stage 0 against the memory as of the previous frame; stage-1 increment"""
        KP, A, nl12, nq = self.KP, self.A, self.nl12, self.nq
        E0, Qin0, Bq0 = self.E0, self.Qin0, self.Bq0
        kcnt, mv = self.cur_cnt.view(-1)[:1], self._tab("mvalid")
        fc = lambda x, i, out: (lambda: ops.linear(x, self.fc_w[i], out, bias=self.fc_b[i], relu=True))
        self._wave_apply(0, "pre", E0, self.B0)
        refs0, m0 = E0[KP:], self.nl0 + self.mem_cap0
        self._attention(self.att_l[0], Qin0[KP:], nl12, refs0, m0, self.ld_0, self.X1[KP:], boxes_q=Bq0[KP:],
                        boxes_k=self.B0[KP:], m_valid=mv[0:1], tail=fc(self.X1[KP:], 1, self.Y1E[KP:nq]))
        self._attention(self.att_l[0], Qin0[:KP], KP, refs0, m0, self.ld_0, self.X1[:KP], boxes_q=Bq0[:KP],
                        boxes_k=self.B0[KP:], m_valid=mv[0:1], n_valid=kcnt, n_valid_off=KP, reuse_kv=True,
                        tail=fc(self.X1[:KP], 1, self.Y1E[:KP]))
        self._wave_pack(1, self.Y1E[KP:KP + A], self.B1[:A])

    def _wave_c(self, im_w, im_h):
        """stage 1; stage-2 increment"""
        KP, A, nl12, nq = self.KP, self.A, self.nl12, self.nq
        Bq0 = self.Bq0
        kcnt, mv = self.cur_cnt.view(-1)[:1], self._tab("mvalid")
        fc = lambda x, i, out: (lambda: ops.linear(x, self.fc_w[i], out, bias=self.fc_b[i], relu=True))
        self._wave_apply(1, "pre", self.Y1E, self.B1)
        m12 = nl12 + self.mem_cap12
        self._attention(self.att_l[1], self.Y1E[KP:nq], nl12, self.Y1E[KP:], m12, self.ld_12, self.X2[KP:],
                        boxes_q=Bq0[KP:], boxes_k=self.B1, m_valid=mv[1:2], tail=fc(self.X2[KP:], 2, self.Y2M[KP:nq]))
        self._attention(self.att_l[1], self.Y1E[:KP], KP, self.Y1E[KP:], m12, self.ld_12, self.X2[:KP],
                        boxes_q=Bq0[:KP], boxes_k=self.B1, m_valid=mv[1:2], n_valid=kcnt, n_valid_off=KP,
                        reuse_kv=True, tail=fc(self.X2[:KP], 2, self.Y2M[:KP]))
        self._wave_pack(2, self.Y2M[KP:KP + A], self.B2[:A])

    def _wave_d(self, im_w, im_h):
        """stage 2, the rest of the group's increments (own frame included: read, then push), G1, predictor, detections"""
        KP = self.KP
        kcnt, mv = self.cur_cnt.view(-1)[:1], self._tab("mvalid")
        self._wave_apply(2, "pre", self.Y2M, self.B2)
        self._stage2(mv)
        self._wave_apply(0, "post", self.E0, self.B0)
        self._wave_apply(1, "post", self.Y1E, self.B1)
        self._wave_apply(2, "post", self.Y2M, self.B2)
        x = self._global_res()
        return self.predict_and_postprocess(x, self.Bq0[:KP], kcnt, im_w, im_h, gemm_done=True)

    def _wave(self, imgs, im_w, im_h, rank, world, payload=None):
        """generator of one wavefront step of rank `rank`: yields (tensor to all-gather, gathered output buffer) four
        times -- frame payloads, then the stage-0 / 1 / 2 memory increments -- and returns the Detections of key frame
        `rank` of the group. `payload`: this rank's frame payload computed elsewhere (tests), instead of `imgs`.
        parallel.drive() runs it over NCCL, parallel.play() over all ranks in one process."""
        self._wave_alloc(world)
        if payload is None:
            with ops.precision(self.cfg.precision):
                self._run_ref(imgs, im_w, im_h)
        else:
            self.payload_in.copy_(payload, non_blocking=True)
        if self.payload_all is None or self.payload_all.shape[0] != world:
            self.payload_all = torch.zeros(world, self.payload_in.numel(), device=self.dev)
        payloads = yield self.payload_in, self.payload_all
        self._wave_fill(rank, world)
        for g in range(rank + 1):                       # the window as of the own key frame
            self._wave_ingest(payloads[g])
        key = (im_w, im_h, rank, world)
        self._wave_seg("a", key, im_w, im_h)
        yield self.w_inc[0], self.w_all[0]
        self._wave_seg("b", key, im_w, im_h)
        yield self.w_inc[1], self.w_all[1]
        self._wave_seg("c", key, im_w, im_h)
        yield self.w_inc[2], self.w_all[2]
        det = self._wave_seg("d", key, im_w, im_h)
        for g in range(rank + 1, world):                # the later frames of the group: state only
            self._wave_ingest(payloads[g])
        return det

    def dist_step_wave(self, imgs, im_w, im_h, group=None):
        """wavefront counterpart of dist_step: returns the Detections of this rank's key frame"""
        import torch.distributed as dist
        from . import parallel
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        return parallel.drive(self._wave(imgs, im_w, im_h, rank, world), group)

    def dist_stepn_wave(self, imgs, im_w, im_h, group=None):
        """n wavefront rounds per call: imgs [2n,3,H,W] = this rank's (local, global) frame pairs of the key frames
        (g * world + rank), g = 0..n-1, of a block of n * world consecutive key frames. The per-frame branch of the n pairs
        runs as ONE batch (like stepn_batched on a single GPU), then the n rounds run in order, each a dist_step_wave on
        its precomputed payload (4 small all-gathers). Returns the n Detections of this rank's key frames (all but the
        last are copies)."""
        import torch.distributed as dist
        from . import parallel
        from .engine import Detections
        world, rank = dist.get_world_size(group), dist.get_rank(group)
        n = imgs.shape[0] // 2
        assert imgs.shape[0] == 2 * n and 1 <= n <= self.MAX_FRAMES_PER_STEP, imgs.shape
        static_in = self.static_input(tuple(imgs.shape))
        if imgs.data_ptr() != static_in.data_ptr():
            static_in.copy_(imgs, non_blocking=True)
        if getattr(self, "payload_n", None) is None:
            self.payload_n = torch.zeros(self.MAX_FRAMES_PER_STEP, self.payload_in.numel(), device=self.dev)
        with ops.precision(self.cfg.precision):
            self._graph_run(("refn", tuple(imgs.shape), im_w, im_h),
                            lambda: self._ref_to_payloads(static_in, im_w, im_h, [self.payload_n[i] for i in range(n)]))
        dets = []
        for g in range(n):
            det = parallel.drive(self._wave(None, im_w, im_h, rank, world, payload=self.payload_n[g]), group)
            if g < n - 1:
                det = Detections(det.boxes.clone(), det.scores.clone(), det.labels.clone(), det.count.clone())
            dets.append(det)
        return dets
