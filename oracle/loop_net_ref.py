"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of how a keyframe from another drone reaches
LoopDetector::on_image_recv (paths relative to /root/reference/swarm_loop/src), with the shipped configuration
(is_pc_replay: false, send_all_features: false):
  * LoopNet::broadcast_fisheye_desc / broadcast_img_desc     loop_net.cpp:20-120 -- one header per direction with
      landmark_num > 0 (feature_num = its flagged landmarks), then one message per landmark with landmarks_flag > 0, in
      index order;
  * on_img_desc_header_recevied / on_landmark_recevied       :196-230, :298-323 -- the receiver rebuilds each image;
  * scan_recv_packets                                        :230-295 -- an image is complete when its landmarks have all
      arrived; landmark_num becomes the number received, and an image without landmarks is never handed on;
  * image_desc_callback                                      :142-172 -- images gathered into a four-direction frame,
      the missing directions null images (generate_null_img_desc);
  * on_image_recv's gates                                    loop_detector.cpp:36-65 -- a foreign frame while
      database_size() == 0, fewer than MIN_DIRECTION_LOOP non-empty directions, landmark_num < MIN_LOOP_NUM.

Two forms:
  * the literal one, at message level: `broadcast` (the sender), `Receiver` (the handlers and the frame assembly) and
    `gate` (on_image_recv).  The frame key is either the image's own msg_id, as image_desc_callback literally keys it
    (random per image, so every multi-direction frame splits into one-direction frames), or the sender's frame_id, the
    evident intent and what the library implements.  Delivery is lossless and in order; with the frame_id key a frame is
    complete when the whole record has been delivered (the reference closes it after 2 * recv_period, or once
    MIN_DIRECTION_LOOP of its images are in).
  * the vectorised one, `receive_record` / `receive_round`: the bytes osb_frontend_receive_dev writes.

Fields the reference's messages do not have travel with the record: its n_dirs and reserved word with the header, and
stereo_match with its landmark.  A record is a numpy structured scalar of RECORD_DTYPE (the bytes of osb_keyframe_record).
"""
from __future__ import annotations

import numpy as np

MAX_DIRS, MAX_KPTS, DEEP, FEAT = 4, 200, 4096, 64
RECORD_DTYPE = np.dtype([("drone_id", "<i4"), ("msg_id", "<i4"), ("n_dirs", "<i4"), ("reserved", "<i4"),
                         ("n_kpts", "<i4", (MAX_DIRS,)), ("n_kpts_down", "<i4", (MAX_DIRS,)),
                         ("global_desc", "<f4", (MAX_DIRS, DEEP)), ("local_desc", "<f4", (MAX_DIRS, MAX_KPTS, FEAT)),
                         ("kpts", "<f4", (MAX_DIRS, MAX_KPTS, 2)), ("stereo_match", "<i4", (MAX_DIRS, MAX_KPTS)),
                         ("landmarks_3d", "<f4", (MAX_DIRS, MAX_KPTS, 3)), ("landmarks_flag", "<i4", (MAX_DIRS, MAX_KPTS))])
RECORD_BYTES = RECORD_DTYPE.itemsize      # 292784


def as_record(b) -> np.ndarray:
    """bytes (or any buffer) of one osb_keyframe_record -> a writable structured scalar"""
    return np.frombuffer(bytearray(bytes(b)), RECORD_DTYPE)[0]


def empty_record() -> np.ndarray:
    return np.zeros((), RECORD_DTYPE)[()]


def dropped(rec) -> np.ndarray:
    """a frame on_image_recv drops: drone_id, msg_id and n_dirs kept, every other field zero"""
    out = empty_record()
    out["drone_id"], out["msg_id"], out["n_dirs"] = rec["drone_id"], rec["msg_id"], rec["n_dirs"]
    return out


# ---- the literal form ----------------------------------------------------------------------------------------------
def broadcast(rec, image_ids):
    """broadcast_fisheye_desc of one record -> the messages in send order: ("header", dict) and ("landmark", dict).
    image_ids[d]: the msg_id broadcast_img_desc draws for direction d (rand() + nsec, :29)."""
    msgs = []
    for d in range(min(max(int(rec["n_dirs"]), 0), MAX_DIRS)):
        n = min(max(int(rec["n_kpts"][d]), 0), MAX_KPTS)
        if n <= 0:                                                     # :22-25
            continue
        flags = rec["landmarks_flag"][d][:n]
        msgs.append(("header", dict(drone_id=int(rec["drone_id"]), frame_id=int(rec["msg_id"]), msg_id=int(image_ids[d]),
                                    direction=d, image_desc=rec["global_desc"][d].copy(),
                                    feature_num=int((flags > 0).sum()),             # :43-48
                                    n_dirs=int(rec["n_dirs"]), reserved=int(rec["reserved"]))))
        for i in range(n):                                             # :68-93
            if flags[i] > 0:
                msgs.append(("landmark", dict(header_id=int(image_ids[d]), landmark_id=i, landmark_2d=rec["kpts"][d][i].copy(),
                                              landmark_3d=rec["landmarks_3d"][d][i].copy(), landmark_flag=int(flags[i]),
                                              feature_descriptor=rec["local_desc"][d][i].copy(),
                                              stereo_match=int(rec["stereo_match"][d][i]))))
    return msgs


class Receiver:
    """LoopNet's receiving side.  key: "frame_id" (the library) or "msg_id" (image_desc_callback as written).
    min_direction_loop: the early frame completion of scan_recv_packets (:276), used with the msg_id key only."""

    def __init__(self, key="frame_id", min_direction_loop=3):
        self.key, self.min_dir = key, min_direction_loop
        self.images, self.active = {}, []                 # received_images, active_receving_msg (in arrival order)
        self.frames, self.active_frames = {}, []          # received_frames, active_receving_frames
        self.delivered = []                               # frame_desc_callback's frames, in order

    def on_header(self, m):                               # :196-228
        img = self.images.setdefault(m["msg_id"], dict(landmarks=[]))
        if m["msg_id"] not in self.active:
            self.active.append(m["msg_id"])
        img.update(m)
        img["landmark_num"] = m["feature_num"]

    def on_landmark(self, m):                             # :298-323
        self.images.setdefault(m["header_id"], dict(landmarks=[]))["landmarks"].append(m)
        self.scan()

    def image_desc_callback(self, img):                   # :142-172
        h = img[self.key]
        if h not in self.frames:
            self.frames[h] = dict(drone_id=img["drone_id"], msg_id=img["frame_id"], n_dirs=img["n_dirs"],
                                  reserved=img["reserved"], images=[None] * MAX_DIRS)
            self.active_frames.append(h)
        self.frames[h]["images"][img["direction"]] = img

    def scan(self, flush=False):                          # scan_recv_packets, :230-295 (no timeouts: lossless delivery)
        done = [i for i in self.active if "feature_num" in self.images[i]
                and self.images[i]["landmark_num"] == len(self.images[i]["landmarks"])]
        for i in done:
            self.active.remove(i)
            img = self.images.pop(i)
            img["landmark_num"] = len(img["landmarks"])
            if img["landmark_num"] > 0:
                self.image_desc_callback(img)
        fin = []
        for h in self.active_frames:
            count = sum(1 for im in self.frames[h]["images"] if im is not None and im["landmark_num"] > 0)
            if flush or (self.key == "msg_id" and count >= self.min_dir):
                fin.append(h)
        for h in fin:
            self.active_frames.remove(h)
            f = self.frames.pop(h)
            f["landmark_num"] = sum(im["landmark_num"] for im in f["images"] if im is not None)
            self.delivered.append(f)

    def receive(self, msgs):
        """the messages of one record, in order; then its frames complete (the timeout of :276 at the latest)"""
        for kind, m in msgs:
            if kind == "header":
                self.on_header(m)
                self.scan()                               # an image without landmarks completes at the next scan
            else:
                self.on_landmark(m)
        self.scan(flush=True)
        out, self.delivered = self.delivered, []
        return out


def gate(frame, self_id, db_rows, min_direction_loop, min_loop_num) -> bool:
    """on_image_recv (loop_detector.cpp:36-65): True when the frame goes on to add_to_database and the query"""
    if frame["drone_id"] != self_id and db_rows == 0:
        return False
    dir_count = sum(1 for im in frame["images"] if im is not None and im["landmark_num"] > 0)
    if dir_count < min_direction_loop:
        return False
    return frame["landmark_num"] >= min_loop_num


def frame_record(frame) -> np.ndarray:
    """a delivered frame in the record layout: direction d's landmarks in arrival order, null images zero with n_kpts 0"""
    out = empty_record()
    out["drone_id"], out["msg_id"], out["n_dirs"], out["reserved"] = (frame["drone_id"], frame["msg_id"], frame["n_dirs"],
                                                                       frame["reserved"])
    out["stereo_match"][:] = -1
    for d in range(min(max(int(frame["n_dirs"]), 0), MAX_DIRS)):
        im = frame["images"][d]
        if im is None or im["landmark_num"] == 0:
            continue
        lms = im["landmarks"]
        out["n_kpts"][d] = len(lms)
        out["global_desc"][d] = im["image_desc"]
        for s, lm in enumerate(lms):
            out["kpts"][d][s] = lm["landmark_2d"]
            out["landmarks_3d"][d][s] = lm["landmark_3d"]
            out["landmarks_flag"][d][s] = lm["landmark_flag"]
            out["local_desc"][d][s] = lm["feature_descriptor"]
            out["stereo_match"][d][s] = lm["stereo_match"]
    return out


def receive_literal(rec, self_id, db_rows, min_direction_loop, min_loop_num, key="frame_id", image_ids=None):
    """one foreign record through broadcast -> Receiver -> gate -> the frames on_image_recv keeps, as records"""
    ids = image_ids if image_ids is not None else [1000 * int(rec["msg_id"]) + d + 1 for d in range(MAX_DIRS)]
    rx = Receiver(key, min_direction_loop)
    frames = rx.receive(broadcast(rec, ids))
    return [frame_record(f) for f in frames if gate(f, self_id, db_rows, min_direction_loop, min_loop_num)]


# ---- the vectorised form -------------------------------------------------------------------------------------------
def receive_record(rec, self_id, db_rows, min_direction_loop, min_loop_num, skipped=False) -> np.ndarray:
    """out_dev[r] of osb_frontend_receive_dev for one record (a structured scalar), db_rows = local + remote store rows"""
    if skipped or int(rec["drone_id"]) == self_id:
        return rec.copy()
    nd = min(max(int(rec["n_dirs"]), 0), MAX_DIRS)
    n = np.clip(rec["n_kpts"], 0, MAX_KPTS)
    keep = (rec["landmarks_flag"] > 0) & (np.arange(MAX_KPTS)[None, :] < n[:, None]) & (np.arange(MAX_DIRS) < nd)[:, None]
    c = keep.sum(axis=1)
    if db_rows == 0 or int((c > 0).sum()) < min_direction_loop or int(c.sum()) < min_loop_num:
        return dropped(rec)
    out = empty_record()
    for f in ("drone_id", "msg_id", "n_dirs", "reserved"):
        out[f] = rec[f]
    out["n_kpts"] = c
    out["stereo_match"][:] = -1
    for d in range(MAX_DIRS):
        idx = np.nonzero(keep[d])[0]
        k = len(idx)
        if k == 0:
            continue
        out["global_desc"][d] = rec["global_desc"][d]
        for f in ("local_desc", "kpts", "stereo_match", "landmarks_3d", "landmarks_flag"):
            out[f][d][:k] = rec[f][d][idx]
    return out


def receive_round(recs, skip, self_id, db_rows, min_direction_loop, min_loop_num) -> list:
    """receive_record for every record of a round (records r == skip copied); gate (a) reads the rows before the round"""
    return [receive_record(r if isinstance(r, np.ndarray) else as_record(r), self_id, db_rows, min_direction_loop,
                           min_loop_num, skipped=(i == skip)) for i, r in enumerate(recs)]
