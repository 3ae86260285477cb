"""Drop-in `configuration` module: same contract as the reference's
configuration.py (reads ./cfg/ape_x.json from the cwd — the path is hard-coded
there, :11 — and lifts its keys to module globals, :39-98), written from
scratch.  Unlike the reference it has no import side effects other than
creating ./weight/<ALG> when missing (checkpoints go there)."""
import json as _json
import os as _os
from datetime import datetime as _dt

_path_ = _os.environ.get("B2RL_CFG", "./cfg/ape_x.json")
with open(_path_) as _f:
    # the reference's cfg files contain no comments; plain JSON is enough
    DATA = _json.load(_f)

ALG = DATA["ALG"]
BASE_PATH = f"./log/{ALG}"
if ALG == "APE_X":
    USE_REWARD_CLIP = DATA.get("USE_REWARD_CLIP", True)
    FRAME_DEDUP = bool(DATA.get("FRAME_DEDUP", False))   # not a reference key: store every distinct frame once
    FRAME_CODEC = bool(DATA.get("FRAME_CODEC", False))   # not a reference key: store that frame pool encoded
    for _k in ("FRAMES_PER_TRANSITION", "DEDUP_WINDOW", "POOL_BYTES_PER_TRANSITION"):
        if _k in DATA:
            globals()[_k] = DATA[_k]
elif ALG == "R2D2":
    FIXED_TRAJECTORY = DATA["FIXED_TRAJECTORY"]
    MEM = DATA["MEM"]
    USE_RESCALING = DATA["USE_RESCALING"]
    FRAME_STRIP = bool(DATA.get("FRAME_STRIP", False))   # not a reference key: store sequences as frame strips
    HOST_FRAMES = bool(DATA.get("HOST_FRAMES", False))   # not a reference key: keep the frames in pinned host memory
    FRAME_DEDUP = bool(DATA.get("FRAME_DEDUP", False))   # not a reference key: store every distinct frame once
    HOST_POOL = bool(DATA.get("HOST_POOL", False))       # not a reference key: keep that frame pool in host memory
    POOL_CODEC = bool(DATA.get("POOL_CODEC", False))     # not a reference key: store that frame pool encoded
    for _k in ("FRAMES_PER_SEQUENCE", "DEDUP_WINDOW", "POOL_BYTES_PER_SEQUENCE"):
        if _k in DATA:
            globals()[_k] = DATA[_k]
elif ALG == "IMPALA":
    C_LAMBDA = DATA["C_LAMBDA"]
    C_VALUE = DATA["C_VALUE"]
    P_VALUE = DATA["P_VALUE"]
    ENTROPY_R = DATA["ENTROPY_R"]
    FRAME_DEDUP = bool(DATA.get("FRAME_DEDUP", False))   # not a reference key: store every distinct frame once
    STAGED_POOL_CODEC = bool(DATA.get("STAGED_POOL_CODEC", False))   # not a reference key: store that pool encoded
    for _k in ("FRAMES_PER_ROLLOUT", "DEDUP_WINDOW", "POOL_BYTES_PER_ROLLOUT"):
        if _k in DATA:
            globals()[_k] = DATA[_k]

use_per = ALG != "IMPALA"
if use_per:
    ALPHA = DATA["ALPHA"]
    BETA = DATA["BETA"]
    TARGET_FREQUENCY = DATA["TARGET_FREQUENCY"]
    N = DATA["N"]

GAMMA = DATA["GAMMA"]
BATCHSIZE = DATA["BATCHSIZE"]
ACTION_SIZE = DATA["ACTION_SIZE"]
UNROLL_STEP = DATA["UNROLL_STEP"]
REPLAY_MEMORY_LEN = DATA["REPLAY_MEMORY_LEN"]
REDIS_SERVER = DATA["REDIS_SERVER"]
REDIS_SERVER_PUSH = DATA.get("REDIS_SERVER_PUSH", "localhost")
DEVICE = DATA["DEVICE"]
LEARNER_DEVICE = DATA["LEARNER_DEVICE"]
BUFFER_SIZE = DATA["BUFFER_SIZE"]
OPTIM_INFO = DATA["optim"]
MODEL = DATA["model"]

CURRENT_TIME = _dt.now().strftime("%m_%d_%Y_%H_%M_%S")
LOG_W = _os.path.join("./weight", ALG, CURRENT_TIME)
