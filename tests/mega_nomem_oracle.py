"""MegaOracle (oracle/mega_oracle.py) without the long-range memory, MODEL.VID.MEGA.MEMORY.ENABLE False: the reference's
_forward_test skips update_memory (roi_box_feature_extractors.py:913-917), so self.mem[i] stays empty after init_memory
and every stage relates its queries to the local rows only. Everything else -- the global stage G0 / G1, the window, the
key frame, the predictor and the post-processing -- is MegaOracle's."""
import mega_oracle as mo


class MegaNoMemOracle(mo.MegaOracle):
    def forward(self, img, infos):
        # MegaOracle.forward reads self.mem[i] before it pushes stage i's rows: emptying the memory on entry leaves
        # every stage of every frame without one (frame 0 re-initialises it itself)
        if infos["frame_category"] != 0:
            self.mem = [None] * self.cfg.stage
            for q in self.mem_q:
                q["rois"].clear()
                q["feats"].clear()
        return super().forward(img, infos)
