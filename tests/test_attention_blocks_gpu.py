"""GPU: the fused attention kernel at token counts around its 192-query block edges, at the model widths (6, 12 and
16 heads) and batch 1, 3 and 8, against the float64 restatement and the error bound of tests/test_depth_kernels_gpu.py.

A CTA owns 192 queries (three consumer warpgroups of 64) and walks the keys in tiles of 128, so the grids below put
NT = ph * pw + 1 at 191, 192 and 193 (NT % 192 = 191, 0, 1) and at 385, 577 and 2443 (DPT-Large at 384 x 384 and
the depth-video size 518 x 924): the last query block is full, holds one row, or ends past NP (NT rounded up to 128),
where its rows would land in the next image's slot of the stacked output if they were written."""
import numpy as np
import pytest

from tests import test_depth_kernels_gpu as T

pytestmark = pytest.mark.gpu


class WideAttnRig(T.AttnRig):
    """T.AttnRig (the last block alone, logits designed key by key) at one of the model widths."""

    def __init__(self, h, w, width):
        T.Rig.__init__(self, *T.REAL[width], h, w, seed=7)
        D, L = self.D, self.L
        for i in range(L):
            self.base[f"l{i}.ls1"] = np.zeros(D, np.float32)
            self.base[f"l{i}.ls2"] = np.zeros(D, np.float32)
        self.base["pe.w"] = (self.base["pe.w"].astype(np.float32) * 0.02).astype(np.float16)
        self.base["pe.b"] = np.zeros(D, np.float32)
        self.base["cls"] = np.zeros(D, np.float32)
        self.base[self.last("ln1.g")] = np.ones(D, np.float32)
        self.base[self.last("ln1.b")] = np.zeros(D, np.float32)
        self.u = np.where(np.arange(D) % 2 == 0, 1.0, -1.0)
        self.restore(*self.base)

    def frames(self, n, seed=0):
        """frames of at least 16 rows (the smallest the engine takes): a 1 x 191 patch grid is a 14-row image, which the
        engine then resizes to; the attention check reads the q, k, v^T the device stored, whatever the pixels were"""
        rng = np.random.default_rng(seed)
        return [rng.integers(0, 256, (max(self.h, 16), self.w, 3), dtype=np.uint8) for _ in range(n)]


# (ph, pw) -> NT: 191, 192, 193, 385, 577, 2443
PEAKED = [((10, 19), "vits"), ((1, 191), "vitb"), ((12, 16), "vitl"), ((16, 24), "vits"), ((24, 24), "vitl"),
          ((37, 66), "vitb")]


@pytest.mark.parametrize("grid,width", PEAKED, ids=[f"{g[0]}x{g[1]}-{w}" for g, w in PEAKED])
def test_attention_block_edges_peaked_softmax(grid, width):
    ph, pw = grid
    rig = WideAttnRig(14 * ph, 14 * pw, width)
    NT, T_ = rig.NT, (rig.NT + 127) // 128
    fr = rig.frames(1)
    tile = np.arange(NT) // 128
    try:
        for key in (5, NT - 1):   # the row maximum far above the runner-up, in the first key tile and on the last key
            off = np.zeros(NT)
            off[key] = 88.0
            rig.design(off, 4.0)
            rig.run(fr)
            lg, _ = T.check_attention(rig, f"attention {ph}x{pw} {rig.H} heads, peak on key {key}")
            top2 = np.sort(lg, axis=1)[:, -2:]
            assert (lg.argmax(axis=1) == key).all() and np.median(top2[:, 1] - top2[:, 0]) > 60
        # the maximum rising tile by tile: the running maximum and the accumulator scale change at every step
        rig.design(min(8.0, 80.0 / max(T_ - 1, 1)) * tile, 1.0)
        rig.run(fr)
        lg, _ = T.check_attention(rig, f"attention {ph}x{pw} {rig.H} heads, maximum rising tile by tile", min_std=0)
        if T_ > 1:
            tmax = np.stack([lg[:, tile == t].max(axis=1) for t in range(T_)], axis=1)
            assert (np.diff(tmax, axis=1) > 0).all(axis=1).mean() > 0.9
        # all logits equal: the mean of v over exactly NT keys
        rig.design(np.zeros(NT), None)
        rig.run(fr)
        lg, _ = T.check_attention(rig, f"attention {ph}x{pw} {rig.H} heads, all logits equal", min_std=0)
        assert not lg.any()
    finally:
        rig.close()


BATCHED = [((10, 19), "vitl", 8), ((1, 191), "vits", 3), ((12, 16), "vitb", 8), ((16, 24), "vitl", 3),
           ((24, 24), "vits", 1), ((37, 66), "vitb", 3)]


@pytest.mark.parametrize("grid,width,B", BATCHED, ids=[f"{g[0]}x{g[1]}-{w}-B{b}" for g, w, b in BATCHED])
def test_attention_block_edges_batch_and_padded_keys(grid, width, B):
    """Every real key ~57 logits below the zero keys of the padded rows [NT, NP) of the images before the last, so that
    one padded key that took part would take all the weight; each image of the batch gives the same bits as that image
    alone, and query rows >= NT (the tail of the last block, past NP when NT % 128 is small) are never written."""
    ph, pw = grid
    rig = WideAttnRig(14 * ph, 14 * pw, width)
    D, NT, NP = rig.D, rig.NT, rig.NP
    try:
        rig.design(np.full(NT, -57.0), 4.0)
        fr = rig.frames(B, seed=4)
        alone = []
        for f in fr:
            rig.run([f])
            alone.append(rig.tok("attn")[:NT].copy())
        if B > 1:
            assert not np.array_equal(alone[0], alone[1])
        rig.run(fr)
        q, k, vt = rig.qkv()
        assert (q[:, :, :NT, 0] == 1).all() and (k[:, :, :NT, 0] < -45).all() and not k[:, :, NT:].any()
        if B > 1:
            assert np.abs(vt[0, :, :, NT:]).max() > 1                  # a padded value is there to be picked up
        T.check_attention(rig, f"attention {ph}x{pw} {rig.H} heads B={B}, padded keys 57 logits above", min_std=0)
        dev = rig.tok("attn").reshape(B, NP, D)
        for i in range(B):
            assert np.array_equal(dev[i, :NT], alone[i]), i
            assert not dev[i, NT:].any(), i
    finally:
        rig.close()
