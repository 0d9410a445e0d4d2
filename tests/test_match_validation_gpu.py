"""The batched BoW entry points reject a vocabulary level or a row capacity that k_build_csr cannot hold in shared memory
((nc + 1 + cap) * 4 > 200 KB) before they enqueue anything: SSLPL_ERR_CAPACITY, no launch counted and every output as the caller left it."""
import numpy as np
import pytest

pytestmark = pytest.mark.gpu
torch = pytest.importorskip("torch")

SMEM_INTS = 200 * 1024 // 4          # MAX_DYN_SMEM in ints
SENTINEL = -7


def _frames(nframes, cap, seed):
    """nframes full frames of cap random descriptors in HBM ([nframes][cap] rows), sslpl_keypoint rows and counts."""
    rng = np.random.default_rng(seed)
    desc = torch.from_numpy(rng.integers(0, 256, (nframes, cap, 32), dtype=np.uint8)).cuda()
    kps = torch.zeros((nframes, cap, 7), dtype=torch.float32, device="cuda")
    n = torch.full((nframes,), cap, dtype=torch.int32, device="cuda")
    return desc, kps, n


def _outputs(nframes, cap):
    d_match = torch.full((nframes - 1, cap), SENTINEL, dtype=torch.int32, device="cuda")
    d_nmatch = torch.full((nframes - 1,), SENTINEL, dtype=torch.int32, device="cuda")
    return d_match, d_nmatch


def test_vocab_level_too_large_for_shared_memory_enqueues_nothing(pkg):
    nframes, cap, levelsup = 2, 64, 0
    parent, ndesc, weight, is_leaf = pkg.Vocabulary.random_arrays(10, 5, seed=3)
    voc = pkg.Vocabulary(10, 5, parent, ndesc, weight, is_leaf)
    nc = voc.level_nodes(levelsup)
    assert nc > SMEM_INTS - cap - 1
    mt = pkg.Matcher(max_features=cap, max_lines=64, max_nodes=nc, max_batch=nframes - 1)
    desc, kps, n = _frames(nframes, cap, 1)
    d_match, d_nmatch = _outputs(nframes, cap)
    d_word = torch.full((nframes, cap), SENTINEL, dtype=torch.int32, device="cuda")
    d_node = torch.full((nframes, cap), SENTINEL, dtype=torch.int32, device="cuda")
    d_weight = torch.full((nframes, cap), float(SENTINEL), dtype=torch.float64, device="cuda")
    before = mt.launch_count
    with pytest.raises(pkg.SslplError, match="error -3:"):
        mt.match_bow_batch_device_vocab(desc.data_ptr(), kps.data_ptr(), n.data_ptr(), nframes, cap, voc, levelsup, 0.7, True,
                                        d_match.data_ptr(), d_nmatch.data_ptr(), d_word.data_ptr(), d_node.data_ptr(), d_weight.data_ptr())
    mt.sync()
    assert mt.launch_count == before
    for t in (d_match, d_nmatch, d_word, d_node, d_weight):
        assert bool((t == SENTINEL).all())


def test_centroids_and_rows_too_large_for_shared_memory_enqueue_nothing(pkg):
    nframes, nc = 2, 6400                       # nc * 32 B fits k_bow_assign's tile; nc + 1 + cap ints do not fit k_build_csr's
    cap = SMEM_INTS - nc                        # = 44,800: nc + 1 + cap exceeds the limit by one
    mt = pkg.Matcher(max_features=cap, max_lines=64, max_nodes=nc, max_batch=nframes - 1)
    desc, kps, n = _frames(nframes, cap, 2)
    cent = torch.from_numpy(np.random.default_rng(4).integers(0, 256, (nc, 32), dtype=np.uint8)).cuda()
    d_match, d_nmatch = _outputs(nframes, cap)
    before = mt.launch_count
    with pytest.raises(pkg.SslplError, match="error -3:"):
        mt.match_bow_batch_device(desc.data_ptr(), kps.data_ptr(), n.data_ptr(), nframes, cap, cent.data_ptr(), nc, 0.7, True,
                                  d_match.data_ptr(), d_nmatch.data_ptr())
    mt.sync()
    assert mt.launch_count == before
    assert bool((d_match == SENTINEL).all()) and bool((d_nmatch == SENTINEL).all())
