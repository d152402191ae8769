"""Time-parallel conversion of an image sequence with the semantics of the reference's video driver.

extra/video_convert.c:226-277 drives ONE `struct CRT` through the whole sequence: blend 0, the field
toggles every frame and the frame parity every other one, output image k is the (never cleared)
output buffer as it stands after field k -- i.e. field k's rows woven into the rows older fields left
behind.  That loop is strictly sequential (its own I/O is synchronous per frame); the only state it
carries from frame to frame is

    rn            the noise LCG        -> closed form: n fields = a jump by n * CRT_INPUT_SIZE steps
    vsync, hsync  where sync was found -> not a function of the image while sync holds: speculated, then
                                          VERIFIED against the predecessor's real final state
    ccf           burst lock           -> re-primed by every crt_modulate (crt_ntsc.c:325-329)
    the output buffer (row weave)      -> a one-frame halo

so the sequence is cut into S segments, each segment is one monitor of a `capi.Batch`, and every step
advances all segments by one frame in a handful of kernel launches.  A segment first decodes the frame
before its first one (the halo) from a speculated sync state; afterwards the speculation is checked:
segment s is exact iff the sync state it holds after its halo equals the state its (exact) predecessor
ended with AND the rows its halo decoded equal the predecessor's last image on those rows.  A segment
that fails the check is simply recomputed from the true state.  The result is bit-identical to the
sequential loop, which tests/test_gpu_video.py checks against the oracle.

Frames shard across ranks the same way (`sharding.shard_range`); the cross-rank check needs the previous
rank's final state and last image, exchanged with one small all_gather.

The VHS build (video_convert.c built with CRT_SYSTEM_NTSCVHS) carries less and one thing more:

    hsync, ccf, rn  -> reset by every crt_modulate (crt_ntscvhs.c:259, 332-336) or overwritten by rand()
                       before use (crt_core.c:349): nothing to carry, and hsync is not compared
    vsync           -> speculated, then verified, as above
    rand() state    -> a pure function of the seed, the frame index and do_aberration (a field's draw count
                       depends on its own draws only): each segment's monitor is seeded and advanced to its
                       first decoded frame with crtx_skip_fields, so it is exact, never speculated

The generator state after a segment's halo is saved, and a repair restores it before redoing the segment.
Each rank computes its own segments' states from the seed, so nothing about rand() is exchanged.
"""
import ctypes as C

from . import capi, layout, sharding

LCG_MUL, LCG_ADD = 214019, 140327895  # crt_core.c:359


def lcg_jump(n):
    """(mul, add) such that n steps of rn = 214019 * rn + 140327895 equal rn * mul + add mod 2^32."""
    am, ac, rm, rc = LCG_MUL, LCG_ADD, 1, 0
    while n:
        if n & 1:
            rc = (rc * am + ac) & 0xFFFFFFFF
            rm = (rm * am) & 0xFFFFFFFF
        ac = (ac * am + ac) & 0xFFFFFFFF
        am = (am * am) & 0xFFFFFFFF
        n >>= 1
    return rm, rc


def _s32(v):
    v &= 0xFFFFFFFF
    return v - (1 << 32) if v & 0x80000000 else v


def frame_parity(f, progressive=False):
    """(field, frame) video_convert.c uses for its f-th processed image (f from 0): lines 261-267."""
    if progressive:
        return 0, 0
    return f & 1, (f >> 1) & 1


class VideoConverter:
    def __init__(self, variant="ntsc", outw=640, outh=480, noise=12, scanlines=1, as_color=1,
                 progressive=False, segments=64, fmt=layout.PIX_BGRA, saturation=10, batch_factory=None, seed=1,
                 do_aberration=0):
        """batch_factory(variant, n) -> an object with capi.Batch's interface (default: capi.Batch itself, the CUDA
        library).  The CPU test-suite injects an oracle-backed stand-in to exercise the scheduling logic below
        (tests/mock_batch.py); nothing else ever should.

        VHS variants only: the sequence is the one srand(seed) followed by video_convert.c's loop gives, with
        do_aberration set in its settings (its -a flag)."""
        import torch
        self.torch = torch
        self._factory = batch_factory if batch_factory is not None else capi.Batch
        self._pool = {}  # monitors are kept between convert() calls: creating and freeing a context costs tens of ms
        self.variant, self.spec = variant, layout.system_spec(variant)
        if self.spec.system not in (layout.SYS_NTSC, layout.SYS_VHS):
            raise ValueError("the video path covers CRT_SYSTEM_NTSC and CRT_SYSTEM_NTSCVHS (what video_convert.c is built for)")
        self.vhs = self.spec.system == layout.SYS_VHS
        self.seed, self.do_aberration = seed, (1 if do_aberration else 0)
        self._extra = dict(do_aberration=self.do_aberration) if self.vhs else {}  # per-field source settings
        self.outw, self.outh, self.noise, self.fmt = outw, outh, noise, fmt
        self.knobs = dict(blend=0, scanlines=scanlines, saturation=saturation)  # video_convert.c:239-241
        self.as_color, self.progressive = as_color, progressive
        self.segments = segments
        self.recomputed = 0  # segments that failed verification in the last convert()

    def _batch(self, n):
        """a context of n monitors, reused across calls (every call sets all of their state; the parts of analog[] no
        crt_modulate writes are zero in a fresh context and stay zero, because this class never varies raw / offsets)"""
        b = self._pool.get(n)
        if b is None:
            b = self._pool[n] = self._factory(self.variant, n)
        return b

    def close(self):
        for b in self._pool.values():
            b.close()
        self._pool = {}

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    # one sequential pass over local frames [lo, hi) on monitor `i` (the repair path)
    def _run_sequential(self, b, i, frames, lo, hi, outputs, first_frame):
        for f in range(lo, hi):
            field, frame = frame_parity(first_frame + f, self.progressive)
            b.set_source(i, frames[f], format=self.fmt, as_color=self.as_color, field=field, frame=frame,
                         raw=0, hue=0, xoffset=0, yoffset=0, **self._extra)
            b.modulate(first=i, count=1)
            b.demodulate(first=i, count=1)
            outputs[f].copy_(self._work[i])

    def convert(self, frames, rn0=194, first_frame=0, group=None):
        """frames: (n, h, w, bpp) uint8 CUDA tensor holding THIS rank's frames [first_frame, first_frame + n)
        of the sequence.  Returns (n, outh, outw, bpp) decoded images, bit-identical to the sequential
        reference loop over the whole sequence (every segment is verified, failures are recomputed)."""
        torch = self.torch
        import torch.distributed as dist
        n = frames.shape[0]
        dev = frames.device
        bpp = layout.bpp4fmt(self.fmt)
        S = max(1, min(self.segments, n))
        spans = [sharding.shard_range(n, s, S) for s in range(S)]  # local frame indices
        b = self._batch(S)
        work_all = torch.zeros(S, self.outh, self.outw, bpp, dtype=torch.uint8, device=dev)
        self._work = [work_all[s] for s in range(S)]  # the monitors' images: one tensor, so a step's images move with one copy
        for s in range(S):
            b.set_monitor(s, self._work[s], fmt=self.fmt, noise=self.noise, **self.knobs)
        b.commit_monitors()
        outputs = torch.empty(n, self.outh, self.outw, bpp, dtype=torch.uint8, device=dev)

        def rn_before(gf):  # LCG state before global frame gf's demodulate (crt_core.c:359, 367)
            m, a = lcg_jump(self.spec.input_size * gf)
            return _s32((rn0 & 0xFFFFFFFF) * m + a)

        # the two frames before this rank's slice (halo of its first segment) live on the previous rank
        world = dist.get_world_size(group) if (dist.is_available() and dist.is_initialized()) else 1
        rank = dist.get_rank(group) if world > 1 else 0
        prev_in = None
        if world > 1:
            counts = torch.tensor([n], dtype=torch.int64, device=dev)
            dist.all_reduce(counts, op=dist.ReduceOp.MIN, group=group)
            if int(counts.item()) < 2:
                raise ValueError("VideoConverter: every rank needs at least 2 frames of the sequence (the two-frame halo of the "
                                 "next rank's first segment); some rank holds %d" % int(counts.item()))
            tails = sharding.allgather_frames(frames[n - 2:n].contiguous(), group)  # (2 * world, h, w, bpp)
            prev_in = tails[2 * (rank - 1):2 * rank] if rank > 0 else None

        def src_frame(gf):
            lf = gf - first_frame
            return frames[lf] if lf >= 0 else prev_in[2 + lf]

        # ---- speculated sync state: what a steady decode holds after a field of each parity (4 probe fields)
        probe = self._batch(1) if S != 1 else self._factory(self.variant, 1)
        scratch = torch.zeros(self.outh, self.outw, bpp, dtype=torch.uint8, device=dev)
        probe.set_monitor(0, scratch, fmt=self.fmt, noise=0, **self.knobs)
        probe.commit_monitors()
        fresh = (capi.State * 1)()  # what crt_init leaves (crt_core.c:250-269): the probe monitor may have been used before
        fresh[0].hsync, fresh[0].vsync, fresh[0].rn = 0, 0, 194
        probe.set_state(fresh)
        if self.vhs:  # the generator the sequence has at this rank's first frame
            probe.seed(self.seed, first=0, count=1)
            probe.skip_fields([first_frame], self.do_aberration)
        after = {}
        for f in range(min(4, n)):
            field, frame = frame_parity(first_frame + f, self.progressive)
            probe.set_source(0, frames[f], format=self.fmt, as_color=self.as_color, field=field, frame=frame, **self._extra)
            probe.modulate()
            probe.demodulate()
            st = probe.get_state()[0]
            after[(first_frame + f) & 1] = (st.hsync, st.vsync)
        if S == 1:
            probe.close()

        # ---- every segment but the sequence's very first decodes a halo of up to two frames first: the
        # output buffer holds rows of the last two fields, so after the halo it must EQUAL the predecessor's
        # last image, which is what gets verified below.
        starts = [first_frame + a for a, _ in spans]
        halo0 = [max(0, g - 2) for g in starts]  # first global frame each segment decodes
        states = (capi.State * S)()
        for s in range(S):
            if halo0[s] == 0:
                hs, vs = 0, 0  # crt_init / crt_reset
            else:
                hs, vs = after.get((halo0[s] - 1) & 1, (0, 0))  # speculation: state after frame halo0 - 1
            states[s].hsync, states[s].vsync, states[s].rn = hs, vs, rn_before(halo0[s])
        b.set_state(states)
        if self.vhs:  # every segment's generator where the sequential loop has it before frame halo0[s]
            b.seed(self.seed, first=0, count=S)
            b.skip_fields(halo0, self.do_aberration)

        # the settings table of the batch as numpy columns (the CUDA library's Batch; the CPU test double has none)
        table = capi.source_table(b.sources) if hasattr(b, "sources") else None
        frame_bytes = frames[0].numel() * frames[0].element_size() if n else 0
        if table is not None:
            import numpy as np
            table["format"], table["as_color"], table["raw"], table["hue"] = self.fmt, self.as_color, 0, 0
            table["xoffset"], table["yoffset"] = 0, 0
            if self.vhs:
                table["do_aberration"] = self.do_aberration
            table["h"], table["w"] = frames.shape[1], frames.shape[2]
            base_mine = frames.data_ptr()
            base_prev = prev_in.data_ptr() if prev_in is not None else 0
            b._keep[("video", 0)] = (frames, prev_in)

        def step(items):  # items: [(segment, global frame)] with contiguous segment indices
            if not items:
                return
            lo_s = min(s for s, _ in items)
            if table is not None:  # whole columns at once: no per-monitor Python work in the step loop
                seg = np.fromiter((s for s, _ in items), dtype=np.int64, count=len(items))
                gf = np.fromiter((g for _, g in items), dtype=np.int64, count=len(items))
                lf = gf - first_frame
                ptr = np.where(lf >= 0, base_mine + lf * frame_bytes, base_prev + (2 + lf) * frame_bytes)
                table["data"][seg] = ptr.astype(np.uint64)
                if self.progressive:
                    table["field"][seg], table["frame"][seg] = 0, 0
                else:
                    table["field"][seg], table["frame"][seg] = gf & 1, (gf >> 1) & 1  # frame_parity
            else:
                for s, gf in items:
                    field, frame = frame_parity(gf, self.progressive)
                    b.set_source(s, src_frame(gf), format=self.fmt, as_color=self.as_color, field=field, frame=frame,
                                 raw=0, hue=0, xoffset=0, yoffset=0, **self._extra)
            b.modulate(first=lo_s, count=len(items))
            b.demodulate(first=lo_s, count=len(items))

        step([(s, starts[s] - 2) for s in range(S) if starts[s] >= 2])
        step([(s, starts[s] - 1) for s in range(S) if starts[s] >= 1])
        st_halo = [(x.hsync, x.vsync) for x in b.get_state()]
        halo_img = {s: self._work[s].clone() for s in range(S) if starts[s] >= 1}
        rand_halo = b.get_rand(0, S) if self.vhs else None  # exact: the halo's draws do not depend on its sync state

        def same_sync(x, y):  # VHS: the next modulate resets hsync, so only vsync carries over
            return x[1] == y[1] if self.vhs else x == y

        # ---- main steps: step t advances every segment still inside its span by one frame; shard_range puts
        # the longer segments first, so the active ones are always 0 .. count-1
        longest = max(e - a for a, e in spans)
        span_lo = torch.tensor([a for a, _ in spans], dtype=torch.int64, device=dev)
        for t in range(longest):
            active = [s for s in range(S) if spans[s][0] + t < spans[s][1]]  # always 0 .. len(active) - 1
            step([(s, starts[s] + t) for s in active])
            outputs.index_copy_(0, span_lo[:len(active)] + t, work_all[:len(active)])  # one copy for the whole step
        finals = [(x.hsync, x.vsync) for x in b.get_state()]

        # ---- verification in sequence order, repairing what the speculation got wrong.  Segment s is exact
        # relative to (pf, pl) = its predecessor's final sync state and last image.  Inside a rank the
        # predecessor is the previous local segment; the first segment of rank r > 0 depends on rank r - 1,
        # whose last segment may itself be repaired -- so ranks repeat "exchange, re-check what the new data
        # invalidates" until a round changes nothing anywhere (at most `world` rounds; one on a single GPU).
        def exchange():
            t_state = torch.tensor([[finals[-1][0], finals[-1][1]]], dtype=torch.int64, device=dev)
            all_state = sharding.allgather_frames(t_state, group)
            all_last = sharding.allgather_frames(outputs[n - 1:n].contiguous(), group)
            if rank == 0:
                return None, None
            return (int(all_state[rank - 1][0]), int(all_state[rank - 1][1])), all_last[rank - 1]

        self.recomputed = 0
        basis = {}       # world > 1: what each checked segment was found exact against
        repaired = set()
        while True:
            prev_final, prev_last = exchange() if world > 1 else (None, None)
            changed = False
            for s in range(S):
                if starts[s] == 0:
                    continue  # began from the true initial state: exact by construction
                pf = finals[s - 1] if s > 0 else prev_final
                pl = outputs[spans[s - 1][1] - 1] if s > 0 else prev_last
                if pf is None:
                    continue
                if s in basis and same_sync(basis[s][0], pf) and bool(torch.equal(basis[s][1], pl)):
                    continue  # already exact against this very predecessor
                if s not in repaired and same_sync(st_halo[s], pf) and bool(torch.equal(halo_img[s], pl)):
                    if world > 1:
                        basis[s] = (pf, pl.clone())
                    continue  # the speculation held
                # redo the segment from the true state and the true image
                self.recomputed += 1
                changed = True
                repaired.add(s)
                if world > 1:
                    basis[s] = (pf, pl.clone())
                a, e = spans[s]
                redo = (capi.State * 1)()
                redo[0].hsync, redo[0].vsync, redo[0].rn = pf[0], pf[1], rn_before(first_frame + a)
                b.set_state(redo, first=s)
                if self.vhs:
                    b.set_rand(rand_halo[s:s + 1], first=s)
                self._work[s].copy_(pl)
                self._run_sequential(b, s, frames, a, e, outputs, first_frame)
                x = b.get_state(first=s, count=1)[0]
                finals[s] = (x.hsync, x.vsync)
            if world == 1:
                break
            flag = torch.tensor([1 if changed else 0], dtype=torch.int64, device=dev)
            dist.all_reduce(flag, op=dist.ReduceOp.MAX, group=group)
            if int(flag.item()) == 0:
                break
        if dev.type == "cuda":
            torch.cuda.synchronize(dev)
        return outputs
