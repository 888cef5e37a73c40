"""The single-frame chain (lm_enqueue -> lm_enqueue_post -> lm_enqueue_pose -> lm_enqueue_pose_nms, then one of
lm_complete / lm_complete_post / lm_complete_pose / lm_complete_detect) and its one completion policy: a frame that kept
more records than the result block holds, or passed more coarse candidates than the candidate list holds (4 Mi entries
up front), is grown and replayed -- refinement, then every later stage enqueued -- in up to three passes, by every
completion alike.

The call-order table runs each sequence of uploads, enqueues and completions on the recorded driver frame and checks
every call's return code, and each output it names against the plain chain of the same frame.  The overflow tests use a
synthetic bank of 1000 small templates with few features at a threshold below 0: every coarse position then passes
and every candidate is kept, so the candidate count is templates x lowest-level positions (frame pixels / 256 at
T = [4, 8]), whatever the frame holds."""
import importlib
import os

import numpy as np
import pytest

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
lib = importlib.import_module("6dpose_b200._lib")
synth = importlib.import_module("6dpose_b200.synth")

CAND_LIST = 4 << 20        # LM_CAND_DEFAULT: candidate-list entries allocated up front
RESULT_BLOCK = 1 << 16     # records of the initial internal result block
THR, TOP_K = 75.0, 3


def code(fn, *args):
    """(return code, output) of a binding call; LM_E_INVALID surfaces as RuntimeError and is not expected here."""
    try:
        return lib.LM_OK, fn(*args)
    except lib.LinemodLibraryError as e:
        return int(str(e).split("error ")[1].split(":")[0]), None


def same(a, b):
    if isinstance(a, dict):
        return a.keys() == b.keys() and all(same(a[k], b[k]) for k in a)
    if isinstance(a, (tuple, list)):
        return len(a) == len(b) and all(same(x, y) for x, y in zip(a, b))
    if isinstance(a, np.ndarray):
        if a.dtype.names:
            return a.shape == b.shape and a.tobytes() == b.tobytes()
        return np.array_equal(a, b, equal_nan=a.dtype.kind == "f")
    return a == b


# ---- call order -----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def driver():
    g = np.load(os.path.join(ROOT, "tests", "golden", "driver_trace.npz"))
    b = np.load(os.path.join(ROOT, "tests", "golden", "bank_allScales_full.npz"))
    packed = dict(class_begin=b["class_begin"], tmeta=b["tmeta"].astype(np.int32), feats=b["feats"].astype(np.int32))
    G = packed["tmeta"].shape[0]
    pose = (g["render"], np.repeat(g["rf0_modelK"][None], G, 0).astype(np.float32),
            np.repeat(g["rf0_modelR"][None], G, 0).astype(np.float32),
            np.repeat(g["rf0_modelT"].reshape(1, 3), G, 0).astype(np.float32))
    rgb, depth = g["rgb"], g["depth"]
    frames = dict(A=(rgb, depth), B=(np.ascontiguousarray(rgb[:, ::-1]), np.ascontiguousarray(depth[:, ::-1])))
    return dict(packed=packed, T=b["T"].tolist(), G=G, pose=pose, sK=g["rf0_sceneK"].astype(np.float32), frames=frames)


def driver_handle(data):
    nat = lib.NativeDetector(data["T"], 0)
    nat.load_bank(data["packed"], 4)
    nat.select(None, 0, 1)
    render, K, R, t = data["pose"]
    nat.set_template_renders(0, [render] * data["G"], K, R, t)
    return nat


def step(nat, data, tok):
    fr, sK = data["frames"], data["sK"]
    ops = dict(
        upA=lambda: nat.upload_images(*fr["A"], None), upB=lambda: nat.upload_images(*fr["B"], None),
        enq=lambda: nat.enqueue(THR), run=lambda: nat.run(THR), post=lambda: nat.enqueue_post(0.5, TOP_K),
        pose=lambda: nat.enqueue_pose(sK, 30, False), pnms=lambda: nat.enqueue_pose_nms(40.0),
        c=nat.complete, cpost=nat.complete_post, cpose=nat.complete_pose, cdet=nat.complete_detect,
        fetch=nat.fetch_records, counters=nat.counters, gate=nat.depth_gate_stats,
        batchA=lambda: nat.detect_batch(fr["A"][0][None], fr["A"][1][None], None, THR, sK[None], 0.5, TOP_K, 30, False, True))
    return code(ops[tok])


# Plain chains of each frame, the references the table's outputs are held to.
REFS = dict(postA="upA enq post cpost", postB="upB enq post cpost", poseA="upA enq post pose cpose",
            poseB="upB enq post pose cpose", detA="upA enq post pose pnms cdet", recA="upA run fetch", cntA="upA run counters")

# Each call in order: `tok` must return LM_OK, `tok!` LM_E_STATE, `tok=ref` LM_OK and the output of REFS[ref]'s last call.
TABLE = [
    # double completion
    ("post completed twice", "upA enq post cpost=postA cpost!"),
    ("pose completed twice", "upA enq post pose cpose=poseA cpose!"),
    ("detect completed twice", "upA enq post pose pnms cdet=detA cdet!"),
    ("lm_complete twice", "upA enq c c fetch=recA counters=cntA"),
    # lm_complete in the middle of a chain
    ("lm_complete inside a post chain", "upA enq post c cpost=postA fetch=recA"),
    ("lm_complete inside a pose chain", "upA enq post pose c cpose=poseA"),
    ("lm_complete inside a detect chain", "upA enq post pose pnms c cdet=detA"),
    # a completion of the wrong stage
    ("lm_complete_post inside a detect chain", "upA enq post pose pnms cpost=postA cdet!"),
    ("lm_complete_post inside a pose chain", "upA enq post pose cpost=postA cpose!"),
    ("lm_complete_pose without a pose stage", "upA enq post cpose! cpost=postA"),
    ("lm_complete_pose with a pose NMS pending", "upA enq post pose pnms cpose! cdet=detA"),
    ("lm_complete_detect without a pose NMS", "upA enq post pose cdet! cpose=poseA"),
    ("lm_complete_post without a post stage", "upA enq cpost!"),
    # pose NMS without a pose stage, and stages out of order
    ("pose NMS without a pose stage", "upA enq post pnms! cpost=postA"),
    ("pose NMS after the pose completed", "upA enq post pose cpose=poseA pnms!"),
    ("pose NMS twice", "upA enq post pose pnms pnms! cdet=detA"),
    ("pose stage without a post stage", "upA enq pose!"),
    ("a new pose stage drops the pending pose NMS", "upA enq post pose pnms pose cpose=poseA"),
    # abandoned chains
    ("new upload before the post completes", "upA enq post upB cpost=postA"),
    ("new upload and chain mid post chain", "upA enq post upB enq post cpost=postB"),
    ("new upload and chain mid pose chain", "upA enq post pose upB enq post pose cpose=poseB"),
    ("lm_enqueue twice", "upA enq enq post cpost=postA"),
    ("lm_enqueue twice inside a post chain", "upA enq post enq cpost=postA"),
    ("a batch abandons the pending pose stage", "upA enq post pose batchA cpose!"),
    # the getters of the completed frame
    ("records before any completion", "upA enq fetch!"),
    ("records after a post completion only", "upA enq post cpost=postA fetch!"),
    ("a new upload drops the completed frame", "upA run upB fetch! counters!"),
    ("lm_enqueue keeps the completed frame's counters", "upA run enq counters=cntA c"),
    ("gate statistics of an ungated frame", "upA run gate!"),
]


@pytest.fixture(scope="module")
def table_handle(driver):
    return driver_handle(driver)


@pytest.fixture(scope="module")
def refs(driver):
    nat = driver_handle(driver)
    out = {}
    for name, seq in REFS.items():
        for tok in seq.split():
            rc, got = step(nat, driver, tok)
            assert rc == lib.LM_OK, (name, tok, rc)
        out[name] = got
    return out


@pytest.mark.parametrize("name,seq", TABLE, ids=[t[0] for t in TABLE])
def test_call_order(driver, refs, table_handle, name, seq):
    nat = table_handle
    for tok in "upA enq post pose pnms cdet".split():   # a clean slate: every stage enqueued and completed
        assert step(nat, driver, tok)[0] == lib.LM_OK
    for tok in seq.split():
        op, _, ref = tok.partition("=")
        rc, got = step(nat, driver, op.rstrip("!"))
        assert rc == (lib.LM_E_STATE if op.endswith("!") else lib.LM_OK), (tok, rc, lib.load().lm_last_error())
        if ref:
            assert same(got, refs[ref]), tok


def test_enqueue_post_on_a_fresh_handle(driver):
    nat = driver_handle(driver)
    nat.upload_images(*driver["frames"]["A"], None)
    assert code(nat.enqueue_post, 0.5, TOP_K)[0] == lib.LM_E_STATE   # no result block before the first lm_enqueue


# ---- overflow ------------------------------------------------------------------------------------------------------
T = [4, 8]
G = 1000
NEG = -1.0                 # every coarse position passes, every candidate is kept


@pytest.fixture(scope="module")
def small():
    bank = synth.synth_bank(G, num_features=8, seed=5, class_ids=("01_template",), size_range=((16, 24), (16, 24)))
    packed = bank.pack(bank.class_ids(), 4)
    render = np.zeros((480, 640), np.uint16)
    render[200:280, 280:360] = 800
    K = np.array([[572.0, 0, 320.0], [0, 572.0, 240.0], [0, 0, 1]], np.float32)
    pose = (render, np.repeat(K[None], G, 0), np.repeat(np.eye(3, dtype=np.float32)[None], G, 0),
            np.repeat(np.array([[0, 0, 800.0]], np.float32), G, 0))
    return dict(bank=bank, packed=packed, pose=pose)


def small_handle(small):
    nat = lib.NativeDetector(T, 0)
    nat.load_bank(small["packed"], 4)
    nat.select(None, 0, 1)
    render, K, R, t = small["pose"]
    nat.set_template_renders(0, [render] * G, K, R, t)
    return nat


def rgbd(W, H, seed=3):
    rng = np.random.default_rng(seed)
    rgb = rng.integers(0, 256, (H, W, 3), dtype=np.uint8)
    depth = (800 + rng.integers(-20, 20, (H, W))).astype(np.uint16)
    sK = np.array([[572.0, 0, W / 2], [0, 572.0, H / 2], [0, 0, 1]], np.float32)
    return rgb, depth, sK


def chains(nat, frame, top_k=TOP_K):
    """The chains a frame can complete through, each returning its outputs with their counts."""
    rgb, depth, sK = frame

    def run():
        nat.upload_images(rgb, depth, None)
        nat.run(NEG)
        c = nat.counters()
        return nat.finish(nat.fetch_records()), c["coarse_candidates"], c["kept"]

    def pose():
        return nat.match_pose(rgb, depth, None, NEG, sK, 0.5, top_k)

    def detect():
        return nat.detect(rgb, depth, None, NEG, sK, 0.5, top_k)

    def post():
        nat.upload_images(rgb, depth, None)
        nat.enqueue(NEG)
        nat.enqueue_post(0.5, top_k)
        return nat.complete_post()
    return dict(run=run, pose=pose, detect=detect, post=post)


def twice(nat, fn, warm=None):
    """fn on a handle whose buffers the frame outgrows, then again on the grown handle: outputs and launch counts."""
    if warm:
        warm()                 # the frame size's first-use work, at a threshold that overflows nothing
    n0 = nat.launch_count()
    first = fn()
    n1 = nat.launch_count()
    second = fn()
    return first, second, n1 - n0, nat.launch_count() - n1


def warm_frame(nat, frame):
    def warm():
        nat.upload_images(frame[0], frame[1], None)
        nat.run(99.9)
    return warm


@pytest.mark.parametrize("path", ["run", "post", "pose", "detect"])
def test_candidate_list_overflow_one_pass(small, path):
    """1280 x 960: 1000 x 4800 candidates, beyond the 4 Mi list but under twice it -- one replay, after which the kept
    count is exact.  About 80 MB of candidate lists and 150 MB of result block (plus as much pinned)."""
    nat = small_handle(small)
    frame = rgbd(1280, 960)
    first, second, launches_first, launches_second = twice(nat, chains(nat, frame)[path], warm_frame(nat, frame))
    assert same(first, second)
    assert launches_first > launches_second                   # the first frame was replayed
    if path == "run":
        assert CAND_LIST < first[1] <= 2 * CAND_LIST and first[2] > RESULT_BLOCK and len(first[0]) > 0


def test_candidate_list_overflow_match_top(small):
    nat = small_handle(small)
    q, _ = synth.synth_frame(1280, 960, levels=2, seed=9, bank=small["bank"], plant=8, T=T)
    nat.match_top(q, 99.9, 0.5, TOP_K)
    n0 = nat.launch_count()
    first = nat.match_top(q, NEG, 0.5, TOP_K)
    n1 = nat.launch_count()
    second = nat.match_top(q, NEG, 0.5, TOP_K)
    assert same(first, second) and first[1] > CAND_LIST
    assert n1 - n0 > nat.launch_count() - n1


def test_candidate_list_overflow_in_a_batch(small):
    """Two equal frames in one lm_detect_batch on a fresh handle: the first is replayed, the second is not."""
    nat = small_handle(small)
    rgb, depth, sK = rgbd(1280, 960)
    args = (np.stack([rgb, rgb]), np.stack([depth, depth]), None, NEG, np.stack([sK, sK]), 0.5, TOP_K, 30, False, True)
    nat.upload_images(rgb, depth, None)
    nat.run(99.9)
    n0 = nat.launch_count()
    got = nat.detect_batch(*args)
    n1 = nat.launch_count()
    assert same(got[0], got[1])
    assert nat.batch_counts[0].tolist() == nat.batch_counts[1].tolist()
    assert nat.batch_counts[0, 3] > CAND_LIST
    again = nat.detect_batch(*args)
    assert same(again, got)
    assert n1 - n0 > nat.launch_count() - n1


@pytest.mark.parametrize("path", ["post", "pose", "detect"])
def test_candidate_list_overflow_two_passes(small, path):
    """1920 x 1280: 1000 x 9600 candidates.  The first pass refines the first 4 Mi of them, so its kept count doubled
    is still too small: a second replay grows the block again.  Device memory: about 150 MB of candidate lists and
    310 MB of result block, and 310 MB pinned."""
    nat = small_handle(small)
    frame = rgbd(1920, 1280)
    first, second, launches_first, launches_second = twice(nat, chains(nat, frame)[path], warm_frame(nat, frame))
    assert same(first, second)
    assert launches_first > launches_second
    records = first[1] if path == "post" else first[4] if path == "pose" else first[4]["records"]
    assert records > 2 * CAND_LIST


def test_external_block_candidate_overflow(small):
    """A caller's result block that holds every record: only the candidate list overflows, and lm_complete_post
    regrows it behind the caller's block as lm_complete does."""
    import torch
    nat = small_handle(small)
    frame = rgbd(1280, 960)
    cap = 5 << 20                                              # records; the frame keeps 1000 x 4800 of them
    block = torch.zeros(16 + 16 * cap, dtype=torch.uint8, device="cuda")
    warm_frame(nat, frame)()
    nat.set_result_buffer(block.data_ptr(), cap)
    post = chains(nat, frame)["post"]
    first = post()
    second = post()
    assert same(first, second) and CAND_LIST < first[1] <= cap
    assert nat.device_result() == (block.data_ptr(), cap)
    nat.set_result_buffer(0, 0)
    del block


def test_complete_then_complete_post_sees_the_grown_frame(small):
    """lm_enqueue, lm_enqueue_post, lm_complete, lm_complete_post on a frame whose records outgrow the result block:
    lm_complete grows the block and replays the box NMS with the refinement, so lm_complete_post returns what the grown
    frame gives -- the next frame's survivors on the same handle -- and not survivors picked from truncated records."""
    nat = small_handle(small)
    q, planted = synth.synth_frame(640, 480, levels=2, seed=21, bank=small["bank"], plant=8, T=T)
    assert planted

    def chain(with_complete):
        nat.upload_quantized(q)
        nat.enqueue(NEG)
        nat.enqueue_post(0.5, 16)
        if with_complete:
            nat.complete()
        return nat.complete_post()
    first = chain(True)
    assert first[1] > RESULT_BLOCK                             # 1000 x 1200 records
    assert same(first, chain(False))
    assert same(first, chain(True))
