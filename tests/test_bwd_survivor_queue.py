"""composite_bwd4.cu: phase B reads each queued splat's record from its survivor-queue slot, so a slot must not be
reused by an append until the splat in it has been drained -- and the drain must find the B4_QUEUE splats it sums, in
replay order, at qbase + h (wrapped).  A restatement of the kernel's queue bookkeeping, run over random hit patterns."""
import numpy as np


def test_backward_queue_keeps_records_until_phase_b_reads_them():
    rng = np.random.default_rng(3)
    for group, queue in ((2, 8), (2, 16), (2, 32), (4, 8), (4, 16), (4, 32), (8, 16)):
        cq = 32 + queue                    # B4_CQ
        assert cq % group == 0
        slots = [None] * cq                # survivor id in a slot; None: free
        head = fill = qpos = qbase = 0
        produced = drained = 0
        for chunk in range(3000):
            hits = int(rng.integers(0, 33)) if chunk % 5 else 32
            for j in range(hits):          # append: slot = head + fill + rank, wrapped once
                slot = head + fill + j
                slot -= cq if slot >= cq else 0
                assert slots[slot] is None, "an append would overwrite a record phase B has not read yet"
                slots[slot] = produced
                produced += 1
            fill += hits
            while fill >= group:           # replay whole groups; the records stay in their slots
                assert head % group == 0 and head + group <= cq
                if qpos == 0:
                    qbase = head
                qpos += group
                if qpos == queue:          # phase B: lane h reads slot qbase + h
                    for h in range(queue):
                        slot = qbase + h if qbase + h < cq else qbase + h - cq
                        assert slots[slot] == drained, "phase B reads the splats in replay order"
                        slots[slot] = None
                        drained += 1
                    qpos = 0
                head = 0 if head + group == cq else head + group
                fill -= group
        assert produced - drained == fill + qpos
