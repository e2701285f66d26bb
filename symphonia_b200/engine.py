"""Engine: one symgpu context (one CUDA device, one stream) driven from Python.

Host entry points take numpy arrays (ideally backed by pinned memory); device entry points take
torch CUDA tensors that already live in HBM.  torch is plumbing only (allocation / pointers).
"""
import ctypes

import numpy as np

from . import _native
from ._native import (AAC_RUN_DTYPE, AAC_TNS_DTYPE, AAC_UNIT_DTYPE, FMT_NUMPY, MP3_GC_DTYPE, MP3_RUN_DTYPE, MPA12_RUN_DTYPE,
                      PCM_SPAN_DTYPE, VORBIS_FLOOR1_DTYPE, VORBIS_RUN_DTYPE, VORBIS_STREAM_DTYPE, VORBIS_STREAM_MC_DTYPE, VORBIS_UNIT_DTYPE,
                      VORBIS_UNIT_MC_DTYPE)


class SymgpuError(RuntimeError):
    def __init__(self, status, detail=""):
        self.status = status
        msg = _native.lib().symgpu_strerror(status).decode()
        super().__init__(f"{msg} [{status}] {detail}".strip())


def _np_ptr(a):
    return a.ctypes.data_as(ctypes.c_void_p)


def _byte_view(data):
    """bytes, or any array, as a contiguous uint8 array."""
    return np.frombuffer(data, dtype=np.uint8) if not isinstance(data, np.ndarray) else np.ascontiguousarray(data, dtype=np.uint8)


def _host_ptr(a):
    """A numpy array's pointer, or None (NULL) for an empty one."""
    return _np_ptr(a) if a.size else None


def _dev_ptr(t):
    """A torch CUDA tensor's pointer, or None (NULL) for an empty one."""
    return ctypes.c_void_p(t.data_ptr()) if t.numel() else None


def file_ranges(ranges):
    """FILE_RANGE_DTYPE records, or (offset, len) pairs, as a contiguous FILE_RANGE_DTYPE array."""
    from ._native import FILE_RANGE_DTYPE
    return np.ascontiguousarray(np.array(ranges, dtype=np.uint64).reshape(-1, 2).view(FILE_RANGE_DTYPE).reshape(-1)
                                if not isinstance(ranges, np.ndarray) or ranges.dtype != FILE_RANGE_DTYPE else ranges)


class Engine:
    def __init__(self, device=0):
        self._lib = _native.lib()
        self._ctx = ctypes.c_void_p()
        st = self._lib.symgpu_ctx_create(int(device), ctypes.byref(self._ctx))
        if st != 0:
            self._ctx = None
            raise SymgpuError(st, "symgpu_ctx_create failed: an H100-class (sm_90) CUDA device is required; "
                                  "there is no CPU fallback")
        self.device = int(device)

    # -- lifetime ---------------------------------------------------------------------------
    def close(self):
        if getattr(self, "_ctx", None):
            self._lib.symgpu_ctx_destroy(self._ctx)
            self._ctx = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def _check(self, st):
        if st != 0:
            raise SymgpuError(st, self._lib.symgpu_last_cuda_error(self._ctx).decode())

    # -- misc -------------------------------------------------------------------------------
    def sync(self):
        self._check(self._lib.symgpu_sync(self._ctx))

    @property
    def cuda_stream(self):
        return self._lib.symgpu_cuda_stream(self._ctx)

    @property
    def numa_node(self):
        """NUMA node the creating thread was bound to by symgpu_ctx_create (-1: unknown, -2: SYMGPU_NUMA_BIND=0)."""
        self._lib.symgpu_ctx_numa_node.restype = ctypes.c_int
        self._lib.symgpu_ctx_numa_node.argtypes = [ctypes.c_void_p]
        return int(self._lib.symgpu_ctx_numa_node(self._ctx))

    @property
    def launch_count(self):
        return int(self._lib.symgpu_launch_count(self._ctx))

    def upload_tables(self, blob):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        self._check(self._lib.symgpu_tables_upload(self._ctx, _np_ptr(blob), blob.nbytes))

    # -- MP3 --------------------------------------------------------------------------------
    def mp3_streams_alloc(self, n_streams):
        self._check(self._lib.symgpu_mp3_streams_alloc(self._ctx, int(n_streams)))

    def mp3_stream_reset(self, stream):
        self._check(self._lib.symgpu_mp3_stream_reset(self._ctx, int(stream)))

    @staticmethod
    def _mp3_args(units, spectra, runs):
        units = np.ascontiguousarray(units, dtype=MP3_GC_DTYPE)
        runs = np.ascontiguousarray(runs, dtype=MP3_RUN_DTYPE)
        n_frames = units.size // 4
        if units.size != n_frames * 4:
            raise ValueError("units must hold 4 granule-channels per frame")
        return units, runs, n_frames

    def mp3_synth_host(self, units, spectra, runs, out=None):
        """units [F,2,2] MP3_GC_DTYPE, spectra [F,2,2,576] f32, runs [R] MP3_RUN_DTYPE -> pcm [F,2,1152]."""
        units, runs, n_frames = self._mp3_args(units, spectra, runs)
        spectra = np.ascontiguousarray(spectra, dtype=np.float32)
        if spectra.size != n_frames * 2304:
            raise ValueError("spectra must be [n_frames, 2, 2, 576]")
        if out is None:
            out = np.empty((n_frames, 2, 1152), dtype=np.float32)
        self._check(self._lib.symgpu_mp3_synth_host(self._ctx, _np_ptr(units), _np_ptr(spectra), _np_ptr(runs),
                                                    len(runs), n_frames, _np_ptr(out)))
        return out

    def mp3_synth_dev(self, units_t, spectra_t, runs, pcm_t):
        """Device-resident variant: torch CUDA tensors (uint8 [F*256], f32 [F,2,2,576], f32 [F,2,1152])."""
        runs = np.ascontiguousarray(runs, dtype=MP3_RUN_DTYPE)
        n_frames = spectra_t.numel() // 2304
        assert units_t.is_cuda and spectra_t.is_cuda and pcm_t.is_cuda
        assert units_t.numel() * units_t.element_size() == n_frames * 256
        assert pcm_t.numel() == n_frames * 2304 and spectra_t.is_contiguous() and pcm_t.is_contiguous()
        self._check(self._lib.symgpu_mp3_synth_dev(self._ctx, ctypes.c_void_p(units_t.data_ptr()),
                                                   ctypes.c_void_p(spectra_t.data_ptr()), _np_ptr(runs), len(runs),
                                                   n_frames, ctypes.c_void_p(pcm_t.data_ptr())))

    def mp3_synth_host_packed(self, units, spectra, runs, fmt, out=None):
        """Like mp3_synth_host, but the output stage runs on the device: returns [F*1152, 2] interleaved
        samples of `fmt` (FMT_*); only those cross PCIe on the way back."""
        units, runs, n_frames = self._mp3_args(units, spectra, runs)
        spectra = np.ascontiguousarray(spectra, dtype=np.float32)
        if spectra.size != n_frames * 2304:
            raise ValueError("spectra must be [n_frames, 2, 2, 576]")
        if out is None:
            out = np.empty((n_frames * 1152, 2), dtype=FMT_NUMPY[fmt])
        self._check(self._lib.symgpu_mp3_synth_host_packed(self._ctx, _np_ptr(units), _np_ptr(spectra), _np_ptr(runs),
                                                           len(runs), n_frames, int(fmt), _np_ptr(out)))
        return out

    def mp3_synth_host_quantized(self, units, quant, runs, fmt=None, out=None):
        """Like mp3_synth_host / mp3_synth_host_packed, fed with the quantised spectra [F,2,2,576] int16 (value =
        sign(q) * |q|^(4/3), looked up on the device).  fmt None: planar f32 [F,2,1152]; else interleaved [F*1152,2]."""
        units, runs, n_frames = self._mp3_args(units, quant, runs)
        quant = np.ascontiguousarray(quant, dtype=np.int16)
        if quant.size != n_frames * 2304:
            raise ValueError("quant must be [n_frames, 2, 2, 576]")
        if out is None:
            out = (np.empty((n_frames, 2, 1152), dtype=np.float32) if fmt is None
                   else np.empty((n_frames * 1152, 2), dtype=FMT_NUMPY[fmt]))
        self._check(self._lib.symgpu_mp3_synth_host_quantized(self._ctx, _np_ptr(units), _np_ptr(quant), _np_ptr(runs),
                                                              len(runs), n_frames, -1 if fmt is None else int(fmt),
                                                              _np_ptr(out)))
        return out

    def mp3_decode_files_host(self, files):
        """EXPERIMENTAL device front-end: files = [(bytes, packets (MPA_PACKET_DTYPE), stream slot)] -> (pcm [F,2,1152],
        good_per_file, frame_of, rounds); only the side-information pass runs on the CPU."""
        from ._native import MP3_FILE_DTYPE, MPA_PACKET_DTYPE
        keep, recs = [], np.zeros(len(files), dtype=MP3_FILE_DTYPE)
        for k, (data, packets, stream) in enumerate(files):
            a = np.frombuffer(data, dtype=np.uint8)
            p = np.ascontiguousarray(packets, dtype=MPA_PACKET_DTYPE)
            keep += [a, p]
            recs[k] = (a.ctypes.data, a.size, p.ctypes.data, len(p), stream, 0)
        total = int(recs["n_packets"].sum())
        pcm = np.zeros((total, 2, 1152), dtype=np.float32)
        good = np.zeros(len(files), dtype=np.uint32)
        frame_of = np.zeros(max(total, 1), dtype=np.uint32)
        rounds = ctypes.c_uint32(0)
        self._check(self._lib.symgpu_mp3_decode_files_host(self._ctx, _np_ptr(recs), len(files), _np_ptr(pcm), total, _np_ptr(good), _np_ptr(frame_of),
                                                           ctypes.byref(rounds)))
        n = int(good.sum())
        return pcm[:n], good, frame_of[:n], rounds.value

    # -- MPEG Layer I / II ---------------------------------------------------------------------
    def mpa12_synth_host(self, subbands, runs, out=None):
        """subbands [F,2,32,n_slots] f32 (n_slots 12: Layer I, 36: Layer II), runs MPA12_RUN_DTYPE -> pcm [F,2,1152]
        (the first 32*n_slots samples of a plane are the frame's PCM).  Uses the MP3 stream state slots."""
        subbands = np.ascontiguousarray(subbands, dtype=np.float32)
        runs = np.ascontiguousarray(runs, dtype=MPA12_RUN_DTYPE)
        n_frames, n_slots = subbands.shape[0], subbands.shape[-1]
        if subbands.shape[1:3] != (2, 32):
            raise ValueError("subbands must be [n_frames, 2, 32, n_slots]")
        if out is None:
            out = np.empty((n_frames, 2, 1152), dtype=np.float32)
        self._check(self._lib.symgpu_mpa12_synth_host(self._ctx, _np_ptr(subbands), _np_ptr(runs), len(runs), n_frames,
                                                      n_slots, _np_ptr(out)))
        return out

    def mpa12_synth_dev(self, subbands_t, runs, n_slots, pcm_t):
        runs = np.ascontiguousarray(runs, dtype=MPA12_RUN_DTYPE)
        n_frames = subbands_t.numel() // (64 * n_slots)
        assert subbands_t.is_cuda and pcm_t.is_cuda and pcm_t.numel() == n_frames * 2304
        self._check(self._lib.symgpu_mpa12_synth_dev(self._ctx, ctypes.c_void_p(subbands_t.data_ptr()), _np_ptr(runs), len(runs),
                                                     n_frames, n_slots, ctypes.c_void_p(pcm_t.data_ptr())))

    # -- FLAC ---------------------------------------------------------------------------------
    def flac_restore_host(self, frames, subframes, samples):
        """In place on `samples` (int32): prediction, wasted-bits shift, channel decorrelation, scaling to 32 bits."""
        from ._native import FLAC_FRAME_DTYPE, FLAC_SUBFRAME_DTYPE
        frames = np.ascontiguousarray(frames, dtype=FLAC_FRAME_DTYPE)
        subframes = np.ascontiguousarray(subframes, dtype=FLAC_SUBFRAME_DTYPE)
        assert samples.dtype == np.int32 and samples.flags.c_contiguous
        self._check(self._lib.symgpu_flac_restore_host(self._ctx, _np_ptr(frames), len(frames), _np_ptr(subframes), len(subframes),
                                                       _np_ptr(samples), samples.size))
        return samples

    def flac_restore_dev(self, frames_t, n_frames, subframes_t, n_subframes, samples_t):
        assert frames_t.is_cuda and subframes_t.is_cuda and samples_t.is_cuda
        self._check(self._lib.symgpu_flac_restore_dev(self._ctx, ctypes.c_void_p(frames_t.data_ptr()), n_frames,
                                                      ctypes.c_void_p(subframes_t.data_ptr()), n_subframes,
                                                      ctypes.c_void_p(samples_t.data_ptr()), samples_t.numel()))

    def flac_decode_host(self, data, jobs, groups, out_cap, out=None, fmt=_native.FMT_S32):
        """Device FLAC decoding of many files in one call: `data` (bytes / uint8 array) holds the packets, jobs FLAC_JOB_DTYPE
        (one per packet, a group's jobs consecutive in stream order), groups FLAC_GROUP_DTYPE (one per file).  Returns (out
        [out_cap] of `fmt`: int32 scaled to 32 bits by default, group_frames uint64 [groups], status uint8 [jobs]); file g's PCM is
        out[out_offset:][:group_frames[g] * channels] as [frames, channels].  A format the library does not know is its to
        refuse (give `out` then)."""
        from ._native import FLAC_GROUP_DTYPE, FLAC_JOB_DTYPE
        a = _byte_view(data)
        jobs = np.ascontiguousarray(jobs, dtype=FLAC_JOB_DTYPE)
        groups = np.ascontiguousarray(groups, dtype=FLAC_GROUP_DTYPE)
        if out is None:
            out = np.zeros(int(out_cap), dtype=FMT_NUMPY[fmt])
        assert out.flags.c_contiguous and out.size >= out_cap and (fmt not in FMT_NUMPY or out.dtype == FMT_NUMPY[fmt])
        group_frames = np.zeros(len(groups), dtype=np.uint64)
        status = np.zeros(len(jobs), dtype=np.uint8)
        self._check(self._lib.symgpu_flac_decode_fmt_host(self._ctx, _host_ptr(a), a.size, _host_ptr(jobs), len(jobs), _host_ptr(groups), len(groups),
                                                          int(fmt), _host_ptr(out), int(out_cap), _host_ptr(group_frames), _host_ptr(status)))
        return out, group_frames, status

    def flac_decode_dev(self, data_t, jobs_t, groups_t, out_t, group_frames_t, status_t, fmt=_native.FMT_S32):
        """Device-resident variant: torch CUDA tensors (uint8 bytes, jobs / groups as uint8 views of the records, out of `fmt`'s
        element type: int32 by default, int64 group_frames, uint8 status); asynchronous on the engine's stream."""
        from ._native import FLAC_GROUP_DTYPE, FLAC_JOB_DTYPE
        ts = (data_t, jobs_t, groups_t, out_t, group_frames_t, status_t)
        assert all(t.is_cuda and t.is_contiguous() for t in ts)
        assert fmt not in FMT_NUMPY or out_t.element_size() == np.dtype(FMT_NUMPY[fmt]).itemsize
        n_jobs = jobs_t.numel() * jobs_t.element_size() // FLAC_JOB_DTYPE.itemsize
        n_groups = groups_t.numel() * groups_t.element_size() // FLAC_GROUP_DTYPE.itemsize
        assert group_frames_t.numel() >= n_groups and group_frames_t.element_size() == 8 and status_t.numel() >= n_jobs
        self._check(self._lib.symgpu_flac_decode_fmt_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _dev_ptr(jobs_t), n_jobs, _dev_ptr(groups_t),
                                                         n_groups, int(fmt), _dev_ptr(out_t), out_t.numel(), _dev_ptr(group_frames_t),
                                                         _dev_ptr(status_t)))

    # -- ALAC ---------------------------------------------------------------------------------
    def alac_decode_host(self, data, jobs, groups, out_cap, out=None, fmt=_native.FMT_S32):
        """Device ALAC decoding of many files in one call: as flac_decode_host, with ALAC_GROUP_DTYPE groups (what each file's
        magic cookie fixes) and FLAC_JOB_DTYPE jobs.  Returns (out, group_frames, status)."""
        from ._native import ALAC_GROUP_DTYPE, FLAC_JOB_DTYPE
        a = _byte_view(data)
        jobs = np.ascontiguousarray(jobs, dtype=FLAC_JOB_DTYPE)
        groups = np.ascontiguousarray(groups, dtype=ALAC_GROUP_DTYPE)
        if out is None:
            out = np.zeros(int(out_cap), dtype=FMT_NUMPY[fmt])
        assert out.flags.c_contiguous and out.size >= out_cap and (fmt not in FMT_NUMPY or out.dtype == FMT_NUMPY[fmt])
        group_frames = np.zeros(len(groups), dtype=np.uint64)
        status = np.zeros(len(jobs), dtype=np.uint8)
        self._check(self._lib.symgpu_alac_decode_fmt_host(self._ctx, _host_ptr(a), a.size, _host_ptr(jobs), len(jobs), _host_ptr(groups), len(groups),
                                                          int(fmt), _host_ptr(out), int(out_cap), _host_ptr(group_frames), _host_ptr(status)))
        return out, group_frames, status

    def alac_decode_dev(self, data_t, jobs_t, groups_t, out_t, group_frames_t, status_t, fmt=_native.FMT_S32):
        """Device-resident variant of alac_decode_host, with the tensors of flac_decode_dev; asynchronous on the engine's stream."""
        from ._native import ALAC_GROUP_DTYPE, FLAC_JOB_DTYPE
        ts = (data_t, jobs_t, groups_t, out_t, group_frames_t, status_t)
        assert all(t.is_cuda and t.is_contiguous() for t in ts)
        assert fmt not in FMT_NUMPY or out_t.element_size() == np.dtype(FMT_NUMPY[fmt]).itemsize
        n_jobs = jobs_t.numel() * jobs_t.element_size() // FLAC_JOB_DTYPE.itemsize
        n_groups = groups_t.numel() * groups_t.element_size() // ALAC_GROUP_DTYPE.itemsize
        assert group_frames_t.numel() >= n_groups and group_frames_t.element_size() == 8 and status_t.numel() >= n_jobs
        self._check(self._lib.symgpu_alac_decode_fmt_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _dev_ptr(jobs_t), n_jobs, _dev_ptr(groups_t),
                                                         n_groups, int(fmt), _dev_ptr(out_t), out_t.numel(), _dev_ptr(group_frames_t),
                                                         _dev_ptr(status_t)))

    # -- many files decoded on the device: one calling convention for MPEG Layer I / II, Layer III, AAC-LC and Vorbis -------------
    def _batch_decode_host(self, fn, lead, dtypes, counted, data, jobs, groups, fmt, out_samples, out):
        """fn(ctx, *lead, bytes, jobs, groups, fmt, out, results, status[, &count]) on host arrays; dtypes: (job, group, result).
        Returns (out, results, status[, count])."""
        job_dtype, group_dtype, result_dtype = dtypes
        a = _byte_view(data)
        jobs = np.ascontiguousarray(jobs, dtype=job_dtype)
        groups = np.ascontiguousarray(groups, dtype=group_dtype)
        if out is None:
            out = np.zeros(int(out_samples), dtype=FMT_NUMPY[fmt])
        assert out.flags.c_contiguous
        results = np.zeros(len(groups), dtype=result_dtype)
        status = np.zeros(len(jobs), dtype=np.uint8)
        count = ctypes.c_uint32(0)
        self._check(fn(self._ctx, *lead, _host_ptr(a), a.size, _host_ptr(jobs), len(jobs), _host_ptr(groups), len(groups), int(fmt),
                       _host_ptr(out), out.nbytes, _host_ptr(results), _host_ptr(status), *([ctypes.byref(count)] if counted else [])))
        return (out, results, status, count.value) if counted else (out, results, status)

    def _batch_decode_dev(self, fn, lead, dtypes, counted, data_t, jobs_t, groups, fmt, out_t, results_t, status_t):
        """fn(ctx, *lead, bytes, jobs, groups, fmt, out, results, status[, &count]) on torch CUDA tensors, `groups` a host array;
        dtypes: (job, group, result).  Returns count, or None."""
        job_dtype, group_dtype, result_dtype = dtypes
        ts = (data_t, jobs_t, out_t, results_t, status_t)
        assert all(t.is_cuda and t.is_contiguous() for t in ts)
        groups = np.ascontiguousarray(groups, dtype=group_dtype)
        n_jobs = jobs_t.numel() * jobs_t.element_size() // job_dtype.itemsize
        assert results_t.numel() * results_t.element_size() >= len(groups) * result_dtype.itemsize and status_t.numel() >= n_jobs
        count = ctypes.c_uint32(0)
        self._check(fn(self._ctx, *lead, _dev_ptr(data_t), data_t.numel(), _dev_ptr(jobs_t), n_jobs, _host_ptr(groups), len(groups), int(fmt),
                       _dev_ptr(out_t), out_t.numel() * out_t.element_size(), _dev_ptr(results_t), _dev_ptr(status_t),
                       *([ctypes.byref(count)] if counted else [])))
        return count.value if counted else None

    def mpa12_decode_host(self, data, jobs, groups, fmt, out_samples, out=None):
        """Device Layer I / II decoding of many files in one call: `data` (bytes / uint8 array) holds the packets, jobs MPA12_JOB_DTYPE
        (one per packet), groups MPA12_GROUP_DTYPE (one per file: its jobs, layer, state slot and output offset).  Returns (out [out_samples]
        of `fmt`, results MPA12_RESULT_DTYPE [groups], status uint8 [jobs]); file g's samples are out[out_offset:][:frames * channels]."""
        from ._native import MPA12_GROUP_DTYPE, MPA12_JOB_DTYPE, MPA12_RESULT_DTYPE
        return self._batch_decode_host(self._lib.symgpu_mpa12_decode_host, (), (MPA12_JOB_DTYPE, MPA12_GROUP_DTYPE, MPA12_RESULT_DTYPE), False,
                                 data, jobs, groups, fmt, out_samples, out)

    def mpa12_decode_dev(self, data_t, jobs_t, groups, fmt, out_t, results_t, status_t):
        """Device-resident variant: torch CUDA tensors (uint8 bytes, jobs / results as uint8 views of the records, `out` of the format's
        element size, uint8 status); `groups` stays a host array.  Asynchronous on the engine's stream."""
        from ._native import MPA12_GROUP_DTYPE, MPA12_JOB_DTYPE, MPA12_RESULT_DTYPE
        self._batch_decode_dev(self._lib.symgpu_mpa12_decode_dev, (), (MPA12_JOB_DTYPE, MPA12_GROUP_DTYPE, MPA12_RESULT_DTYPE), False,
                         data_t, jobs_t, groups, fmt, out_t, results_t, status_t)

    def mp3_decode_host(self, data, jobs, groups, fmt, out_samples, out=None):
        """Device Layer III decoding of many files in one call: `data` (bytes / uint8 array) holds the packets, jobs MP3_JOB_DTYPE (one per
        packet), groups MP3_GROUP_DTYPE (one per file: its jobs, granules, channels, state slot and output offset).  Returns (out
        [out_samples] of `fmt`, results MP3_RESULT_DTYPE [groups], status uint8 [jobs], rounds); file g's samples are
        out[out_offset:][:frames * channels]."""
        from ._native import MP3_GROUP_DTYPE, MP3_JOB_DTYPE, MP3_RESULT_DTYPE
        return self._batch_decode_host(self._lib.symgpu_mp3_decode_host, (), (MP3_JOB_DTYPE, MP3_GROUP_DTYPE, MP3_RESULT_DTYPE), True,
                                 data, jobs, groups, fmt, out_samples, out)

    def mp3_decode_dev(self, data_t, jobs_t, groups, fmt, out_t, results_t, status_t):
        """Device-resident variant: torch CUDA tensors (uint8 bytes, jobs / results as uint8 views of the records, `out` of the format's
        element size, uint8 status); `groups` stays a host array.  Waits for the engine's stream once per round (a 4-byte flag); the
        synthesis and the output stage are left queued on it.  Returns the number of rounds."""
        from ._native import MP3_GROUP_DTYPE, MP3_JOB_DTYPE, MP3_RESULT_DTYPE
        return self._batch_decode_dev(self._lib.symgpu_mp3_decode_dev, (), (MP3_JOB_DTYPE, MP3_GROUP_DTYPE, MP3_RESULT_DTYPE), True,
                                data_t, jobs_t, groups, fmt, out_t, results_t, status_t)

    def aac_decode_host(self, data, jobs, groups, fmt, out_samples, out=None):
        """Device AAC-LC decoding of many files in one call: `data` (bytes / uint8 array) holds the raw_data_blocks, jobs PIECE_DTYPE
        (one per packet), groups AAC_GROUP_DTYPE (one per file: its jobs, sample rate, channels, state slot and output offset).
        Returns (out [out_samples] of `fmt`, results AAC_RESULT_DTYPE [groups], status uint8 [jobs], n_redecoded); file g's samples
        are out[out_offset:][:frames * channels]."""
        from ._native import AAC_GROUP_DTYPE, AAC_RESULT_DTYPE, PIECE_DTYPE
        return self._batch_decode_host(self._lib.symgpu_aac_decode_host, (), (PIECE_DTYPE, AAC_GROUP_DTYPE, AAC_RESULT_DTYPE), True,
                                 data, jobs, groups, fmt, out_samples, out)

    def aac_decode_dev(self, data_t, jobs_t, groups, fmt, out_t, results_t, status_t):
        """Device-resident variant: torch CUDA tensors (uint8 bytes, jobs / results as uint8 views of the records, `out` of the format's
        element size, uint8 status); `groups` stays a host array.  Waits for the engine's stream for one 8-byte readback (and once
        more when pulses need the host); the synthesis and the output stage are left queued on it.  Returns n_redecoded."""
        from ._native import AAC_GROUP_DTYPE, AAC_RESULT_DTYPE, PIECE_DTYPE
        return self._batch_decode_dev(self._lib.symgpu_aac_decode_dev, (), (PIECE_DTYPE, AAC_GROUP_DTYPE, AAC_RESULT_DTYPE), True,
                                data_t, jobs_t, groups, fmt, out_t, results_t, status_t)

    @staticmethod
    def _vorbis_setup_args(headers, setups):
        """The leading arguments of symgpu_vorbis_decode_host / _dev: the header bytes and the setups that name them."""
        from ._native import VORBIS_SETUP_REF_DTYPE
        h = _byte_view(headers)
        setups = np.ascontiguousarray(setups, dtype=VORBIS_SETUP_REF_DTYPE)
        return _host_ptr(h), h.size, _host_ptr(setups), len(setups)   # (a numpy pointer keeps its array alive)

    def vorbis_decode_host(self, headers, setups, data, jobs, groups, fmt, out_samples, out=None):
        """Device Ogg Vorbis decoding of many files in one call: `headers` (bytes) holds the identification / setup packets that
        `setups` (VORBIS_SETUP_REF_DTYPE, one per distinct pair) name, `data` the audio packets, jobs VORBIS_JOB_DTYPE (one per
        packet, with the reader's discard / end trim), groups VORBIS_GROUP_DTYPE (one per file: its jobs, setup and output
        offset).  Returns (out [out_samples] of `fmt`, results VORBIS_RESULT_DTYPE [groups], status uint8 [jobs]); file g's
        samples are out[out_offset:][:frames * channels].  Replaces the engine's Vorbis stream and floor registration."""
        from ._native import VORBIS_GROUP_DTYPE, VORBIS_JOB_DTYPE, VORBIS_RESULT_DTYPE
        return self._batch_decode_host(self._lib.symgpu_vorbis_decode_host, self._vorbis_setup_args(headers, setups),
                                 (VORBIS_JOB_DTYPE, VORBIS_GROUP_DTYPE, VORBIS_RESULT_DTYPE), False, data, jobs, groups, fmt, out_samples, out)

    def vorbis_decode_dev(self, headers, setups, data_t, jobs_t, groups, fmt, out_t, results_t, status_t):
        """Device-resident variant: torch CUDA tensors (uint8 bytes, jobs / results as uint8 views of the records, `out` of the
        format's element size, uint8 status); `headers`, `setups` and `groups` stay on the host.  The host waits only for the
        stream / floor registration; the decode, the synthesis and the output stage are left queued on the engine's stream."""
        from ._native import VORBIS_GROUP_DTYPE, VORBIS_JOB_DTYPE, VORBIS_RESULT_DTYPE
        self._batch_decode_dev(self._lib.symgpu_vorbis_decode_dev, self._vorbis_setup_args(headers, setups),
                         (VORBIS_JOB_DTYPE, VORBIS_GROUP_DTYPE, VORBIS_RESULT_DTYPE), False, data_t, jobs_t, groups, fmt, out_t, results_t, status_t)

    # -- Ogg pages indexed on the device --------------------------------------------------------
    def ogg_index_dev(self, data_t, ranges, cap_packets=None, cap_pieces=None):
        """(packets_t, pieces_t, index) for the files data_t[offset : offset + len] of `ranges` (FILE_RANGE_DTYPE records, or
        (offset, len) pairs) in a uint8 CUDA tensor: packets_t / pieces_t the uint8 bytes of OGG_PACKET_DTYPE / PIECE_DTYPE
        records on the device, index the files' OGG_FILE_INDEX_DTYPE records on the host.  File i's tables, its packets
        [first_packet, first_packet + n_packets) and pieces likewise, equal packetizer.ogg_index of its bytes.  Without
        capacities the sizes are found first by a call with none (its index read back), then the tables written by a second."""
        import torch
        from ._native import OGG_FILE_INDEX_DTYPE
        assert data_t.is_cuda and data_t.is_contiguous() and data_t.dtype == torch.uint8
        r = file_ranges(ranges)
        index_t = torch.empty(len(r) * OGG_FILE_INDEX_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)

        def call(packets_t, pieces_t):
            torch.cuda.current_stream(data_t.device).synchronize()  # data_t and the outputs are torch's: written / allocated on its stream
            self.ogg_index_dev_queue(data_t, r, packets_t, pieces_t, index_t)
            self.sync()
            return index_t.cpu().numpy().view(OGG_FILE_INDEX_DTYPE)

        def totals(ix):
            return (int(ix["first_packet"][-1]) + int(ix["n_packets"][-1]), int(ix["first_piece"][-1]) + int(ix["n_pieces"][-1])) if len(ix) else (0, 0)
        none = torch.empty(0, dtype=torch.uint8, device=data_t.device)
        if cap_packets is None or cap_pieces is None:
            cap_packets, cap_pieces = totals(call(none, none))
        packets_t = torch.empty(cap_packets * _native.OGG_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
        pieces_t = torch.empty(cap_pieces * _native.PIECE_DTYPE.itemsize, dtype=torch.uint8, device=data_t.device)
        return packets_t, pieces_t, call(packets_t, pieces_t)

    def ogg_index_dev_queue(self, data_t, ranges, packets_t, pieces_t, index_t):
        """symgpu_ogg_index_dev on uint8 CUDA tensors (packets_t / pieces_t / index_t the bytes of their records), left queued on
        the engine's stream: no wait for torch's stream before it, none for the engine's after it."""
        from ._native import OGG_PACKET_DTYPE, PIECE_DTYPE
        r = file_ranges(ranges)
        self._check(self._lib.symgpu_ogg_index_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                   packets_t.numel() // OGG_PACKET_DTYPE.itemsize, _dev_ptr(pieces_t),
                                                   pieces_t.numel() // PIECE_DTYPE.itemsize, _dev_ptr(index_t)))

    def _index_dev(self, queue, data_t, ranges, cap, min_frame, per_cap, per_file):
        """Allocate, queue, wait and read back, for a device index whose queue(data_t, ranges, cap, *tables, *records) writes
        `cap` records of each dtype of per_cap (None: that table is not written) and one record per file of each dtype of
        per_file.  cap=None: the lengths // min_frame, summed.  Returns the tables, on the device, and the records, read back.
        adts_index_dev, mpa_index_dev, flac_index_dev and the device-files decoders of decode.py index through it."""
        import torch
        assert data_t.is_cuda and data_t.is_contiguous() and data_t.dtype == torch.uint8
        r = file_ranges(ranges)
        if cap is None:
            cap = int((r["len"] // min_frame).sum())
        d = data_t.device
        kept = [None if dt is None else torch.empty(cap * dt.itemsize, dtype=torch.uint8, device=d) for dt in per_cap]
        read = [torch.empty(len(r) * dt.itemsize, dtype=torch.uint8, device=d) for dt in per_file]
        torch.cuda.current_stream(d).synchronize()  # data_t and the outputs are torch's: written / allocated on its stream
        queue(data_t, r, cap, *kept, *read)
        self.sync()
        return (*kept, *(t.cpu().numpy().view(dt) for t, dt in zip(read, per_file)))

    # -- CAF holding ALAC indexed on the device ----------------------------------------------------
    def caf_index_dev(self, data_t, ranges):
        """(infos, first_packet, packets_t, jobs_t, read_back_bytes) for the CAF files data_t[offset : offset + len] of `ranges`
        (FILE_RANGE_DTYPE records, or (offset, len) pairs) in a uint8 CUDA tensor: infos the files' CAF_INFO_DTYPE records and
        first_packet their uint64 starts, on the host; packets_t / jobs_t the uint8 bytes of CAF_PACKET_DTYPE / FLAC_JOB_DTYPE
        records on the device, room for every file's table_packets.  File i's info and packets, [first_packet, first_packet +
        n_packets), equal packetizer.caf_index of its bytes; its jobs are what alac_decode_dev takes (group i).  read_back_bytes
        counts the two reads of the infos and the one of first_packet."""
        import torch
        from ._native import CAF_INFO_DTYPE, CAF_PACKET_DTYPE, FLAC_JOB_DTYPE
        assert data_t.is_cuda and data_t.is_contiguous() and data_t.dtype == torch.uint8
        r = file_ranges(ranges)
        n, d = len(r), data_t.device
        infos_t = torch.empty(n * CAF_INFO_DTYPE.itemsize, dtype=torch.uint8, device=d)
        first_t = torch.empty(n * 8, dtype=torch.uint8, device=d)
        torch.cuda.current_stream(d).synchronize()  # data_t and the outputs are torch's: written / allocated on its stream
        self._check(self._lib.symgpu_caf_open_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), n, _dev_ptr(infos_t)))
        self.sync()
        heads = infos_t.cpu().numpy().view(CAF_INFO_DTYPE)
        cap = int(heads["table_packets"][heads["open"] == 0].astype(np.int64).sum())
        packets_t = torch.empty(max(cap, 1) * CAF_PACKET_DTYPE.itemsize, dtype=torch.uint8, device=d)
        jobs_t = torch.empty(max(cap, 1) * FLAC_JOB_DTYPE.itemsize, dtype=torch.uint8, device=d)
        torch.cuda.current_stream(d).synchronize()
        self._check(self._lib.symgpu_caf_packets_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), n, _dev_ptr(infos_t),
                                                     _dev_ptr(first_t), _dev_ptr(packets_t), _dev_ptr(jobs_t), cap))
        self.sync()
        infos = infos_t.cpu().numpy().view(CAF_INFO_DTYPE)
        first = first_t.cpu().numpy().view(np.uint64)
        return infos, first, packets_t, jobs_t, heads.nbytes + infos.nbytes + first.nbytes

    # -- ADTS frames indexed on the device ---------------------------------------------------------
    def adts_index_dev(self, data_t, ranges, cap=None):
        """(packets_t, jobs_t, index) for the files data_t[offset : offset + len] of `ranges` (FILE_RANGE_DTYPE records, or
        (offset, len) pairs) in a uint8 CUDA tensor: packets_t / jobs_t the uint8 bytes of `cap` ADTS_PACKET_DTYPE / PIECE_DTYPE
        records on the device, index the files' ADTS_FILE_INDEX_DTYPE records on the host.  File i's packets, [first_packet,
        first_packet + n_packets), equal packetizer.adts_index of its bytes, with its stop; its jobs are the same payloads as
        byte ranges of data_t.  cap=None: the lengths // 7, summed, which every file fits (a frame is at least 7 bytes)."""
        from ._native import ADTS_FILE_INDEX_DTYPE, ADTS_PACKET_DTYPE, PIECE_DTYPE
        return self._index_dev(self.adts_index_dev_queue, data_t, ranges, cap, 7, (ADTS_PACKET_DTYPE, PIECE_DTYPE), (ADTS_FILE_INDEX_DTYPE,))

    def adts_index_dev_queue(self, data_t, ranges, cap, packets_t, jobs_t, index_t):
        """symgpu_adts_index_dev on uint8 CUDA tensors (packets_t / jobs_t, either None, holding `cap` records; index_t one record
        per file), left queued on the engine's stream after the call's one wait: no wait for torch's stream before it."""
        from ._native import ADTS_PACKET_DTYPE, PIECE_DTYPE
        r = file_ranges(ranges)
        assert packets_t is None or packets_t.numel() >= cap * ADTS_PACKET_DTYPE.itemsize
        assert jobs_t is None or jobs_t.numel() >= cap * PIECE_DTYPE.itemsize
        self._check(self._lib.symgpu_adts_index_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r),
                                                    None if packets_t is None else _dev_ptr(packets_t),
                                                    None if jobs_t is None else _dev_ptr(jobs_t), cap, _dev_ptr(index_t)))

    # -- MPEG audio frames indexed on the device ---------------------------------------------------------
    def mpa_index_dev(self, data_t, ranges, cap=None, seekable=True):
        """(packets_t, jobs_t, index, tracks) for the files data_t[offset : offset + len] of `ranges` (FILE_RANGE_DTYPE records, or
        (offset, len) pairs) in a uint8 CUDA tensor: packets_t / jobs_t the uint8 bytes of `cap` MPA_PACKET_DTYPE / MP3_JOB_DTYPE
        records on the device, index the files' MPA_FILE_INDEX_DTYPE records and tracks their MPA_TRACK_DTYPE records on the host.
        File i's track and packets, [first_packet, first_packet + n_packets), equal packetizer.mpa_index(bytes, seekable) (status
        MPA_NO_FRAME where that raises); its jobs are the same frames as byte ranges of data_t.  cap=None: the lengths // 24, summed,
        which every file fits (a frame is at least 24 bytes)."""
        from ._native import MP3_JOB_DTYPE, MPA_FILE_INDEX_DTYPE, MPA_MIN_FRAME, MPA_PACKET_DTYPE, MPA_TRACK_DTYPE
        return self._index_dev(lambda *args: self.mpa_index_dev_queue(*args, seekable), data_t, ranges, cap, MPA_MIN_FRAME,
                               (MPA_PACKET_DTYPE, MP3_JOB_DTYPE), (MPA_FILE_INDEX_DTYPE, MPA_TRACK_DTYPE))

    def mpa_index_dev_queue(self, data_t, ranges, cap, packets_t, jobs_t, index_t, tracks_t, seekable=True):
        """symgpu_mpa_index_dev on uint8 CUDA tensors (packets_t / jobs_t, either None, holding `cap` records; index_t and tracks_t
        one record per file), left queued on the engine's stream after the call's one wait: no wait for torch's stream before it."""
        from ._native import MP3_JOB_DTYPE, MPA_PACKET_DTYPE
        r = file_ranges(ranges)
        assert packets_t is None or packets_t.numel() >= cap * MPA_PACKET_DTYPE.itemsize
        assert jobs_t is None or jobs_t.numel() >= cap * MP3_JOB_DTYPE.itemsize
        self._check(self._lib.symgpu_mpa_index_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), int(bool(seekable)),
                                                   None if packets_t is None else _dev_ptr(packets_t),
                                                   None if jobs_t is None else _dev_ptr(jobs_t), cap, _dev_ptr(index_t), _dev_ptr(tracks_t)))

    # -- native FLAC frames indexed on the device ---------------------------------------------------------
    def flac_index_dev(self, data_t, ranges, cap=None):
        """(packets_t, jobs_t, index, infos) for the native FLAC files data_t[offset : offset + len] of `ranges` (FILE_RANGE_DTYPE
        records, or (offset, len) pairs) in a uint8 CUDA tensor: packets_t / jobs_t the uint8 bytes of `cap` FLAC_PACKET_DTYPE /
        FLAC_JOB_DTYPE records on the device, index the files' FLAC_FILE_INDEX_DTYPE records and infos their FLAC_STREAM_INFO_DTYPE
        records on the host.  File i's info and packets, [first_packet, first_packet + n_packets), equal packetizer.flac_index of its
        bytes (index["open"] the status where that raises, its info zeros); its jobs are the same frames as byte ranges of data_t,
        group i, slot = dur.  cap=None: the lengths // 8, summed, which every file fits (a frame is at least 8 bytes)."""
        from ._native import FLAC_FILE_INDEX_DTYPE, FLAC_JOB_DTYPE, FLAC_MIN_FRAME, FLAC_PACKET_DTYPE, FLAC_STREAM_INFO_DTYPE
        return self._index_dev(self.flac_index_dev_queue, data_t, ranges, cap, FLAC_MIN_FRAME, (FLAC_PACKET_DTYPE, FLAC_JOB_DTYPE),
                               (FLAC_FILE_INDEX_DTYPE, FLAC_STREAM_INFO_DTYPE))

    def flac_index_dev_queue(self, data_t, ranges, cap, packets_t, jobs_t, index_t, infos_t):
        """symgpu_flac_index_dev on uint8 CUDA tensors (packets_t / jobs_t, either None, holding `cap` records; index_t and infos_t
        one record per file), left queued on the engine's stream after the call's one wait: no wait for torch's stream before it."""
        from ._native import FLAC_JOB_DTYPE, FLAC_PACKET_DTYPE
        r = file_ranges(ranges)
        assert packets_t is None or packets_t.numel() >= cap * FLAC_PACKET_DTYPE.itemsize
        assert jobs_t is None or jobs_t.numel() >= cap * FLAC_JOB_DTYPE.itemsize
        self._check(self._lib.symgpu_flac_index_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r),
                                                    None if packets_t is None else _dev_ptr(packets_t),
                                                    None if jobs_t is None else _dev_ptr(jobs_t), cap, _dev_ptr(index_t), _dev_ptr(infos_t)))

    # -- Vorbis jobs built on the device from the device Ogg index (uint8 CUDA tensors holding the records; queued, no wait) -----
    def vorbis_heads_dev(self, data_t, ranges, packets_t, pieces_t, index_t, heads_t, ranks_t):
        """symgpu_vorbis_heads_dev: per file a VORBIS_FILE_HEADS_DTYPE record in heads_t, per packet of packets_t a
        VORBIS_PACKET_RANK_DTYPE record in ranks_t, from the tables ogg_index_dev_queue wrote."""
        from ._native import OGG_PACKET_DTYPE
        r = file_ranges(ranges)
        self._check(self._lib.symgpu_vorbis_heads_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                      packets_t.numel() // OGG_PACKET_DTYPE.itemsize, _dev_ptr(pieces_t), _dev_ptr(index_t),
                                                      _dev_ptr(heads_t), _dev_ptr(ranks_t)))

    def ogg_gather_dev(self, data_t, ranges, packets_t, pieces_t, index_t, refs, out_t):
        """symgpu_ogg_gather_dev: the packets `refs` (OGG_PACKET_REF_DTYPE, host) name copied to out_t[dst ..]."""
        from ._native import OGG_PACKET_REF_DTYPE
        r = file_ranges(ranges)
        refs = np.ascontiguousarray(refs, dtype=OGG_PACKET_REF_DTYPE)
        self._check(self._lib.symgpu_ogg_gather_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                    _dev_ptr(pieces_t), _dev_ptr(index_t), _host_ptr(refs), len(refs), _dev_ptr(out_t), out_t.numel()))

    def vorbis_jobs_dev(self, data_t, ranges, packets_t, pieces_t, index_t, ranks_t, file_jobs, out_t, jobs_t):
        """symgpu_vorbis_jobs_dev: every audio packet of the files whose VORBIS_FILE_JOBS_DTYPE record (host) has n_modes gathered
        to out_t, and its VORBIS_JOB_DTYPE record written to jobs_t."""
        from ._native import OGG_PACKET_DTYPE, VORBIS_FILE_JOBS_DTYPE, VORBIS_JOB_DTYPE
        r = file_ranges(ranges)
        file_jobs = np.ascontiguousarray(file_jobs, dtype=VORBIS_FILE_JOBS_DTYPE)
        self._check(self._lib.symgpu_vorbis_jobs_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                     packets_t.numel() // OGG_PACKET_DTYPE.itemsize, _dev_ptr(pieces_t), _dev_ptr(index_t),
                                                     _dev_ptr(ranks_t), _host_ptr(file_jobs), _dev_ptr(out_t), out_t.numel(), _dev_ptr(jobs_t),
                                                     jobs_t.numel() // VORBIS_JOB_DTYPE.itemsize))

    # -- FLAC-in-Ogg jobs built on the device from the device Ogg index (uint8 CUDA tensors holding the records; queued, no wait) -
    def ogg_flac_heads_dev(self, data_t, ranges, packets_t, pieces_t, index_t, group_of, heads_t, ranks_t):
        """symgpu_ogg_flac_heads_dev: per group (group_of, host uint32 per file, OGG_FLAC_NO_GROUP for a file left out) an
        OGG_FLAC_FILE_DTYPE record in heads_t, per packet of packets_t an OGG_FLAC_PACKET_RANK_DTYPE record in ranks_t, from the
        tables ogg_index_dev_queue wrote."""
        from ._native import OGG_FLAC_FILE_DTYPE, OGG_PACKET_DTYPE
        r = file_ranges(ranges)
        group_of = np.ascontiguousarray(group_of, dtype=np.uint32)
        assert len(group_of) == len(r)
        self._check(self._lib.symgpu_ogg_flac_heads_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                        packets_t.numel() // OGG_PACKET_DTYPE.itemsize, _dev_ptr(pieces_t), _dev_ptr(index_t),
                                                        _host_ptr(group_of), heads_t.numel() // OGG_FLAC_FILE_DTYPE.itemsize, _dev_ptr(heads_t),
                                                        _dev_ptr(ranks_t)))

    def ogg_flac_jobs_dev(self, data_t, ranges, packets_t, pieces_t, index_t, group_of, ranks_t, out_t, jobs_t):
        """symgpu_ogg_flac_jobs_dev: every audio packet's bytes gathered to out_t and its FLAC_JOB_DTYPE record (group from
        group_of) written to jobs_t, from the ranks ogg_flac_heads_dev wrote."""
        from ._native import FLAC_JOB_DTYPE, OGG_PACKET_DTYPE
        r = file_ranges(ranges)
        group_of = np.ascontiguousarray(group_of, dtype=np.uint32)
        assert len(group_of) == len(r)
        self._check(self._lib.symgpu_ogg_flac_jobs_dev(self._ctx, _dev_ptr(data_t), data_t.numel(), _host_ptr(r), len(r), _dev_ptr(packets_t),
                                                       packets_t.numel() // OGG_PACKET_DTYPE.itemsize, _dev_ptr(pieces_t), _dev_ptr(index_t),
                                                       _host_ptr(group_of), _dev_ptr(ranks_t), _dev_ptr(out_t), out_t.numel(), _dev_ptr(jobs_t),
                                                       jobs_t.numel() // FLAC_JOB_DTYPE.itemsize))

    # -- output stage -------------------------------------------------------------------------
    def pcm_pack_host(self, pcm, spans, channels, fmt, out_frames, plane_stride=0, frames=0, n_spans=None, out=None):
        """Trim + interleave + convert planar f32 `pcm` (any shape, flat indexing) into [out_frames, channels]
        samples.  spans: PCM_SPAN_DTYPE array, or None for uniform packets (plane_stride, frames, n_spans)."""
        pcm = np.ascontiguousarray(pcm, dtype=np.float32)
        if spans is not None:
            spans = np.ascontiguousarray(spans, dtype=PCM_SPAN_DTYPE)
            n_spans = len(spans)
        if out is None:
            out = np.zeros((out_frames, channels), dtype=FMT_NUMPY[fmt])
        self._check(self._lib.symgpu_pcm_pack_host(self._ctx, _np_ptr(pcm), pcm.size,
                                                   _np_ptr(spans) if spans is not None else None, n_spans, channels,
                                                   plane_stride, frames, int(fmt), _np_ptr(out), out.nbytes))
        return out

    def pcm_pack_dev(self, pcm_t, spans_t, n_spans, channels, fmt, out_t, plane_stride=0, frames=0):
        """Device-resident variant (torch CUDA tensors; spans_t may be None for uniform packets)."""
        assert pcm_t.is_cuda and out_t.is_cuda
        self._check(self._lib.symgpu_pcm_pack_dev(self._ctx, ctypes.c_void_p(pcm_t.data_ptr()),
                                                  ctypes.c_void_p(spans_t.data_ptr()) if spans_t is not None else None,
                                                  n_spans, channels, plane_stride, frames, int(fmt),
                                                  ctypes.c_void_p(out_t.data_ptr())))

    # -- AAC --------------------------------------------------------------------------------
    def aac_streams_alloc(self, n_streams):
        self._check(self._lib.symgpu_aac_streams_alloc(self._ctx, int(n_streams)))

    def aac_stream_reset(self, stream):
        self._check(self._lib.symgpu_aac_stream_reset(self._ctx, int(stream)))

    def aac_synth_host(self, units, tns, coeffs, runs, out=None):
        """units [F,2] AAC_UNIT_DTYPE, tns [T] AAC_TNS_DTYPE, coeffs [F,2,1024] f32 -> pcm [F,2,1024]."""
        units = np.ascontiguousarray(units, dtype=AAC_UNIT_DTYPE)
        tns = np.ascontiguousarray(tns, dtype=AAC_TNS_DTYPE)
        runs = np.ascontiguousarray(runs, dtype=AAC_RUN_DTYPE)
        coeffs = np.ascontiguousarray(coeffs, dtype=np.float32)
        n_frames = units.size // 2
        if coeffs.size != n_frames * 2048:
            raise ValueError("coeffs must be [n_frames, 2, 1024]")
        if out is None:
            out = np.empty((n_frames, 2, 1024), dtype=np.float32)
        self._check(self._lib.symgpu_aac_synth_host(self._ctx, _np_ptr(units), _np_ptr(tns) if len(tns) else None, len(tns),
                                                    _np_ptr(coeffs), _np_ptr(runs), len(runs), n_frames, _np_ptr(out)))
        return out

    def aac_synth_dev(self, units_t, tns_t, n_tns, coeffs_t, runs, pcm_t):
        runs = np.ascontiguousarray(runs, dtype=AAC_RUN_DTYPE)
        n_frames = coeffs_t.numel() // 2048
        self._check(self._lib.symgpu_aac_synth_dev(
            self._ctx, ctypes.c_void_p(units_t.data_ptr()), ctypes.c_void_p(tns_t.data_ptr()) if n_tns else None, int(n_tns),
            ctypes.c_void_p(coeffs_t.data_ptr()), _np_ptr(runs), len(runs), n_frames, ctypes.c_void_p(pcm_t.data_ptr())))

    # -- Vorbis -----------------------------------------------------------------------------
    def vorbis_streams_set(self, streams):
        streams = np.ascontiguousarray(streams, dtype=VORBIS_STREAM_DTYPE)
        self._check(self._lib.symgpu_vorbis_streams_set(self._ctx, _np_ptr(streams), len(streams)))

    def vorbis_floors_set(self, floors):
        floors = np.ascontiguousarray(floors, dtype=VORBIS_FLOOR1_DTYPE)
        self._check(self._lib.symgpu_vorbis_floors_set(self._ctx, _np_ptr(floors), len(floors)))

    def vorbis_stream_reset(self, stream):
        self._check(self._lib.symgpu_vorbis_stream_reset(self._ctx, int(stream)))

    def vorbis_synth_host(self, units, floor_y, residue, runs, slot, out=None):
        """units [P] VORBIS_UNIT_DTYPE, floor_y [P,2,65] u16, residue [P,2,slot] f32 -> pcm [P,2,slot]."""
        units = np.ascontiguousarray(units, dtype=VORBIS_UNIT_DTYPE)
        floor_y = np.ascontiguousarray(floor_y, dtype=np.uint16)
        residue = np.ascontiguousarray(residue, dtype=np.float32)
        runs = np.ascontiguousarray(runs, dtype=VORBIS_RUN_DTYPE)
        n = len(units)
        if residue.size != n * 2 * slot or floor_y.size != n * 130:
            raise ValueError("residue must be [n, 2, slot] and floor_y [n, 2, 65]")
        if out is None:
            out = np.empty((n, 2, slot), dtype=np.float32)
        self._check(self._lib.symgpu_vorbis_synth_host(self._ctx, _np_ptr(units), _np_ptr(floor_y), _np_ptr(residue),
                                                       _np_ptr(runs), len(runs), n, int(slot), _np_ptr(out)))
        return out

    def vorbis_mc_streams_set(self, streams):
        """Multichannel Vorbis streams (up to 8 channels, every coupling step of the mapping): VORBIS_STREAM_MC_DTYPE records."""
        streams = np.ascontiguousarray(streams, dtype=VORBIS_STREAM_MC_DTYPE)
        self._check(self._lib.symgpu_vorbis_mc_streams_set(self._ctx, _np_ptr(streams), len(streams)))

    def vorbis_mc_synth_host(self, units, floor_y, residue, runs, channels, slot, out=None):
        """units [P] VORBIS_UNIT_MC_DTYPE, floor_y [P,C,65] u16, residue [P,C,slot] f32 -> pcm [P,C,slot]."""
        units = np.ascontiguousarray(units, dtype=VORBIS_UNIT_MC_DTYPE)
        floor_y = np.ascontiguousarray(floor_y, dtype=np.uint16)
        residue = np.ascontiguousarray(residue, dtype=np.float32)
        runs = np.ascontiguousarray(runs, dtype=VORBIS_RUN_DTYPE)
        n, C = len(units), int(channels)
        if residue.size != n * C * slot or floor_y.size != n * C * 65:
            raise ValueError("residue must be [n, channels, slot] and floor_y [n, channels, 65]")
        if out is None:
            out = np.empty((n, C, slot), dtype=np.float32)
        self._check(self._lib.symgpu_vorbis_mc_synth_host(self._ctx, _np_ptr(units), _np_ptr(floor_y), _np_ptr(residue), _np_ptr(runs), len(runs), n,
                                                          C, int(slot), _np_ptr(out)))
        return out

    def vorbis_synth_dev(self, units_t, floor_y_t, residue_t, runs, slot, pcm_t):
        runs = np.ascontiguousarray(runs, dtype=VORBIS_RUN_DTYPE)
        n = units_t.numel() * units_t.element_size() // 16
        self._check(self._lib.symgpu_vorbis_synth_dev(
            self._ctx, ctypes.c_void_p(units_t.data_ptr()), ctypes.c_void_p(floor_y_t.data_ptr()),
            ctypes.c_void_p(residue_t.data_ptr()), _np_ptr(runs), len(runs), n, int(slot), ctypes.c_void_p(pcm_t.data_ptr())))

    # -- thread-safe submission: many decoder threads, one context, shared launches ---------------------------------------
    # Every submit copies one frame into the context's open batch and returns a ticket; wait returns that frame's PCM, running
    # the batch if no other thread has.  ctypes releases the GIL around both, so Python threads can share one Engine.
    def _submit(self, fn, *args):
        ticket = _native.Ticket()
        self._check(fn(self._ctx, *args, ctypes.byref(ticket)))
        return ticket

    def _wait(self, fn, ticket, out):
        self._check(fn(self._ctx, ticket, _np_ptr(out)))
        return out

    def mp3_submit(self, stream, units, spectra, granules_per_frame=2, channels=2):
        """units [2,2] MP3_GC_DTYPE, spectra [2,2,576] f32 of one frame -> ticket."""
        units = np.ascontiguousarray(units, dtype=MP3_GC_DTYPE)
        spectra = np.ascontiguousarray(spectra, dtype=np.float32)
        if units.size != 4 or spectra.size != 2304:
            raise ValueError("one frame: units [2,2], spectra [2,2,576]")
        return self._submit(self._lib.symgpu_mp3_submit, int(stream), _np_ptr(units), _np_ptr(spectra), int(granules_per_frame), int(channels))

    def mp3_wait(self, ticket, out=None):
        return self._wait(self._lib.symgpu_mp3_wait, ticket, np.empty((2, 1152), dtype=np.float32) if out is None else out)

    def aac_submit(self, stream, units, tns, coeffs, channels=2):
        """units [2] AAC_UNIT_DTYPE (tns_first counted from the start of `tns`), tns [T] AAC_TNS_DTYPE, coeffs [2,1024] f32 -> ticket."""
        units = np.ascontiguousarray(units, dtype=AAC_UNIT_DTYPE)
        tns = np.ascontiguousarray(tns, dtype=AAC_TNS_DTYPE)
        coeffs = np.ascontiguousarray(coeffs, dtype=np.float32)
        if units.size != 2 or coeffs.size != 2048:
            raise ValueError("one frame: units [2], coeffs [2,1024]")
        return self._submit(self._lib.symgpu_aac_submit, int(stream), _np_ptr(units), _np_ptr(tns) if len(tns) else None, len(tns),
                            _np_ptr(coeffs), int(channels))

    def aac_wait(self, ticket, out=None):
        """pcm [2,1024] of the ticket's frame."""
        return self._wait(self._lib.symgpu_aac_wait, ticket, np.empty((2, 1024), dtype=np.float32) if out is None else out)

    def mpa12_submit(self, stream, subbands, channels=2):
        """subbands [2,32,n_slots] f32 of one Layer I (n_slots 12) or Layer II (36) frame; `stream` is an MP3 state slot -> ticket."""
        subbands = np.ascontiguousarray(subbands, dtype=np.float32)
        if subbands.shape[:2] != (2, 32) or subbands.ndim != 3:
            raise ValueError("one frame: subbands [2,32,n_slots]")
        return self._submit(self._lib.symgpu_mpa12_submit, int(stream), _np_ptr(subbands), subbands.shape[2], int(channels))

    def mpa12_wait(self, ticket, out=None):
        """pcm [2,1152]; plane(ch)[:32 * n_slots] is the frame's output."""
        return self._wait(self._lib.symgpu_mpa12_wait, ticket, np.empty((2, 1152), dtype=np.float32) if out is None else out)

    def vorbis_streams_alloc(self, n_streams):
        """Reserves n Vorbis stream slots, configured one at a time with vorbis_stream_configure."""
        self._check(self._lib.symgpu_vorbis_streams_alloc(self._ctx, int(n_streams)))

    def vorbis_stream_configure(self, stream, config, floors):
        """config: one VORBIS_STREAM_DTYPE record, floors [<= 64] VORBIS_FLOOR1_DTYPE -> floor_base (= 64 * stream): what a unit's
        floor index of this stream is counted from."""
        config = np.ascontiguousarray(config, dtype=VORBIS_STREAM_DTYPE).reshape(1)
        floors = np.ascontiguousarray(floors, dtype=VORBIS_FLOOR1_DTYPE)
        base = ctypes.c_uint32(0)
        self._check(self._lib.symgpu_vorbis_stream_configure(self._ctx, int(stream), _np_ptr(config), _np_ptr(floors) if len(floors) else None,
                                                             len(floors), ctypes.byref(base)))
        return base.value

    def vorbis_submit(self, stream, unit, floor_y, residue):
        """unit VORBIS_UNIT_DTYPE (floors counted from the slot's floor_base), floor_y [2,65] u16, residue [2,slot] f32 -> ticket."""
        unit = np.ascontiguousarray(unit, dtype=VORBIS_UNIT_DTYPE).reshape(1)
        floor_y = np.ascontiguousarray(floor_y, dtype=np.uint16)
        residue = np.ascontiguousarray(residue, dtype=np.float32)
        if floor_y.size != 130 or residue.ndim != 2 or residue.shape[0] != 2:
            raise ValueError("one packet: floor_y [2,65], residue [2,slot]")
        return self._submit(self._lib.symgpu_vorbis_submit, int(stream), _np_ptr(unit), _np_ptr(floor_y), _np_ptr(residue), residue.shape[1])

    def vorbis_wait(self, ticket, slot, out=None):
        """pcm [2,slot] with the slot the packet was submitted with."""
        return self._wait(self._lib.symgpu_vorbis_wait, ticket, np.empty((2, int(slot)), dtype=np.float32) if out is None else out)

    def async_stats(self, codec):
        """(launch batches, frames they held) of the queue of `codec` (_native.CODEC_*)."""
        b, f = ctypes.c_uint64(0), ctypes.c_uint64(0)
        self._check(self._lib.symgpu_async_stats(self._ctx, int(codec), ctypes.byref(b), ctypes.byref(f)))
        return b.value, f.value
