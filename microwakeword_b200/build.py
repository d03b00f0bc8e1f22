"""Build libmww_b200.so in-tree with nvcc for sm_90a (no JIT cache: the .so travels with the repo
snapshot to the GPU box).  `python -m microwakeword_b200.build` or `__graft_entry__.build()`."""

from __future__ import annotations

import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libmww_b200.so")
SOURCES = ["mww_capi.cu", "mww_detector_capi.cu", "mww_verify_capi.cu", "mww_endpoint_capi.cu", "mww_media_guard_capi.cu", "mww_playback_capi.cu", "mww_frontend.cu", "mww_nn.cu", "mww_nn_int8.cu", "mww_nn_live.cu", "mww_nn_i8_live.cu", "mww_nn_generic.cu", "mww_nn_tc.cu", "mww_streams.cu", "mww_records.cu", "mww_detect.cu", "mww_tables.cc", "mww_container.cc"]
# the input-rate resampler kernel (mww_set_input_rate) is a companion library that libmww_b200.so links (rpath $ORIGIN): the
# main library's own kernel set stays the one the SASS fixtures under tests/golden/ record
RS_OUT = os.path.join(HERE, "libmww_resample.so")
RS_SOURCES = ["mww_resample.cu"]
# the same kernel on one rate's members of a tile (per-stream rates, mww_set_stream_rates), likewise apart, so that
# libmww_resample.so keeps the two instantiations a handle with one input rate runs
RR_OUT = os.path.join(HERE, "libmww_resample_rates.so")
RR_SOURCES = ["mww_resample_rates.cu"]
# likewise the streaming detector's kernels (mww_detector_*)
DET_OUT = os.path.join(HERE, "libmww_detector.so")
DET_SOURCES = ["mww_detector.cu"]
# and the multi-model detector's (mww_multi_detector_create), so that libmww_detector.so keeps the plain detector's three
MD_OUT = os.path.join(HERE, "libmww_detector_models.so")
MD_SOURCES = ["mww_detector_models.cu"]
# and both detectors' per-row-cutoff kernels (mww_set_detector_cutoffs, mww_set_multi_detector_cutoffs), so that those two
# libraries keep exactly the kernels uniform mode runs
DC_OUT = os.path.join(HERE, "libmww_detector_cutoffs.so")
DC_SOURCES = ["mww_detector_cutoffs.cu"]
# and the frontend and resampler kernels for G.711 audio (mww_features_g711 and the other _g711 entry points), so that
# libmww_b200.so and the two resampler libraries keep exactly the kernels int16 and float32 audio run
G711_OUT = os.path.join(HERE, "libmww_g711.so")
G711_SOURCES = ["mww_frontend_g711.cu"]
# and the audio history's kernels (mww_set_audio_history), so that a handle without a history runs exactly the kernels it ran
HIST_OUT = os.path.join(HERE, "libmww_history.so")
HIST_SOURCES = ["mww_history.cu"]
# and the detector records' kernels (mww_export_detector_rows / mww_import_detector_rows), so that libmww_b200.so and the three
# detector libraries keep exactly the kernels they had
DR_OUT = os.path.join(HERE, "libmww_detector_records.so")
DR_SOURCES = ["mww_detector_records.cu"]
# and second-stage verification's two kernels (mww_verify_streams / mww_verify_detections), so that every library above keeps
# exactly the kernels it had
VER_OUT = os.path.join(HERE, "libmww_verify.so")
VER_SOURCES = ["mww_verify.cu"]
# and the endpointer's four kernels (mww_endpointer_*), likewise
EP_OUT = os.path.join(HERE, "libmww_endpoint.so")
EP_SOURCES = ["mww_endpoint.cu"]
# and the kernels that move a stream's serving state between handles: the audio history write (mww_write_audio_history) and
# the endpointer records (mww_export_endpointer_rows / mww_import_endpointer_rows), so that libmww_history.so and
# libmww_endpoint.so keep exactly the kernels they had
SR_OUT = os.path.join(HERE, "libmww_serving_records.so")
SR_SOURCES = ["mww_serving_records.cu"]
# and the kernels of event positions: the timed detectors' updates, the history read that ends at given positions
# (mww_read_audio_history_at) and the verifier slots that end at their events (mww_verify_detections_at), so that the detector,
# history, endpoint and verify libraries keep exactly the kernels they had
EVP_OUT = os.path.join(HERE, "libmww_event_positions.so")
EVP_SOURCES = ["mww_event_positions.cu"]
# and the kernels of grouped detection: the grouped timed updates and the close of every group (mww_group_detector_events), so
# that every library above keeps exactly the kernels it had
GRP_OUT = os.path.join(HERE, "libmww_detector_groups.so")
GRP_SOURCES = ["mww_detector_groups.cu"]
# and the media guard's four kernels (mww_media_guard_create and the checks), likewise
MG_OUT = os.path.join(HERE, "libmww_media_guard.so")
MG_SOURCES = ["mww_media_guard.cu"]
# and the playback guard's three kernels (mww_playback_guard_create and the writes, reads and checks), likewise
PB_OUT = os.path.join(HERE, "libmww_playback.so")
PB_SOURCES = ["mww_playback.cu"]
# and group arbitration's kernels (mww_arbitrate_detector_groups): the arbitrated timed updates and their close, likewise
ARB_OUT = os.path.join(HERE, "libmww_group_arbitration.so")
ARB_SOURCES = ["mww_group_arbitration.cu"]
# and the persistent fused clip frontend (k1_clip_kernel, every sample type), which every long call with enough streams runs, so
# that libmww_b200.so and libmww_g711.so keep exactly the kernels they had
FC_OUT = os.path.join(HERE, "libmww_frontend_clip.so")
FC_SOURCES = ["mww_frontend_clip.cu"]
# and the resampler on members whose rows each hold their own sample format (mww_set_stream_formats, the _mixed entry points),
# so that libmww_resample_rates.so and libmww_g711.so keep exactly the kernels they had
RM_OUT = os.path.join(HERE, "libmww_resample_mixed.so")
RM_SOURCES = ["mww_resample_mixed.cu"]
# and the positioned endpointer's kernels (mww_endpointer_arm_at and the forms that keep each row's mute word), so that
# libmww_endpoint.so and libmww_serving_records.so keep exactly the kernels they had
EPA_OUT = os.path.join(HERE, "libmww_endpoint_at.so")
EPA_SOURCES = ["mww_endpoint_at.cu"]
NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17", "-shared",
         "-Xcompiler", "-fPIC", "-cudart", "static"]


STAMP = OUT + ".srchash"


def source_hash() -> str:
    """sha256 over every file of csrc/, include/mww.h and the compiler flags: what the binary was built from.  Content, not
    mtimes -- the tree is copied to the GPU box, where timestamps mean nothing."""
    import hashlib
    h = hashlib.sha256(" ".join(FLAGS).encode())
    deps = sorted(os.path.join(CSRC, f) for f in os.listdir(CSRC)) + [os.path.join(os.path.dirname(HERE), "include", "mww.h")]
    for d in deps:
        h.update(os.path.basename(d).encode())
        with open(d, "rb") as f:
            h.update(f.read())
    return h.hexdigest()


def _stale() -> bool:
    if not all(os.path.exists(p) for p in (OUT, RS_OUT, RR_OUT, DET_OUT, MD_OUT, DC_OUT, G711_OUT, HIST_OUT, DR_OUT, VER_OUT, EP_OUT, SR_OUT, EVP_OUT, GRP_OUT, MG_OUT, PB_OUT, ARB_OUT, FC_OUT, RM_OUT, EPA_OUT, STAMP)):
        return True
    try:
        return open(STAMP).read().strip() != source_hash()
    except OSError:
        return True


def build(force: bool = False, verbose: bool = False) -> str:
    if not force and not _stale():
        return OUT
    if not os.path.exists(NVCC):
        raise RuntimeError("nvcc not found at %s; libmww_b200.so must be prebuilt (there is no CPU fallback)" % NVCC)
    import fcntl
    with open(OUT + ".lock", "w") as lock:               # several ranks may arrive here at once: one builds, the rest wait
        fcntl.flock(lock, fcntl.LOCK_EX)
        if not force and not _stale():
            return OUT
        for out, sources, extra in ((RS_OUT, RS_SOURCES, []), (RR_OUT, RR_SOURCES, []), (DET_OUT, DET_SOURCES, []),
                                    (MD_OUT, MD_SOURCES, []), (DC_OUT, DC_SOURCES, []), (G711_OUT, G711_SOURCES, []),
                                    (HIST_OUT, HIST_SOURCES, []), (DR_OUT, DR_SOURCES, []), (VER_OUT, VER_SOURCES, []),
                                    (EP_OUT, EP_SOURCES, []), (SR_OUT, SR_SOURCES, []), (EVP_OUT, EVP_SOURCES, []),
                                    (GRP_OUT, GRP_SOURCES, []), (MG_OUT, MG_SOURCES, []), (PB_OUT, PB_SOURCES, []),
                                    (ARB_OUT, ARB_SOURCES, []), (FC_OUT, FC_SOURCES, []), (RM_OUT, RM_SOURCES, []),
                                    (EPA_OUT, EPA_SOURCES, []),
                                    (OUT, SOURCES, ["-L" + HERE, "-lmww_resample", "-lmww_resample_rates", "-lmww_detector",
                                                    "-lmww_detector_models", "-lmww_detector_cutoffs", "-lmww_g711", "-lmww_history",
                                                    "-lmww_detector_records", "-lmww_verify", "-lmww_endpoint", "-lmww_serving_records",
                                                    "-lmww_event_positions", "-lmww_detector_groups", "-lmww_media_guard", "-lmww_playback",
                                                    "-lmww_group_arbitration", "-lmww_frontend_clip", "-lmww_resample_mixed", "-lmww_endpoint_at",
                                                    "-Xlinker", "-rpath,$ORIGIN"])):
            tmp = out + ".tmp.%d" % os.getpid()
            cmd = [NVCC] + FLAGS + (["-Xptxas", "-v"] if verbose else []) + ["-o", tmp] + [os.path.join(CSRC, s) for s in sources] + extra
            res = subprocess.run(cmd, capture_output=True, text=True)
            if res.returncode != 0:
                sys.stderr.write(res.stdout + res.stderr)
                if os.path.exists(tmp):
                    os.unlink(tmp)
                raise RuntimeError("nvcc failed building %s" % os.path.basename(out))
            if verbose:
                sys.stderr.write(res.stderr)
            os.replace(tmp, out)                           # a process that has the old file mapped keeps its own copy
        with open(STAMP, "w") as f:
            f.write(source_hash() + "\n")
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
