"""`uncalled index`, `uncalled map` and `uncalled sim` (reference scripts/uncalled:38-78,127-167 with the options of
uncalled/args.py:87-161,218-286) on this package: same sub-commands, option names, defaults, stderr progress
lines and PAF output.  `python -m uncalled_b200 map <prefix> <fast5s...>`.  `--device` picks the GPU of this
process; under `torchrun --nproc-per-node N -m uncalled_b200 map ...` every rank maps its share of the fast5 files on
its own GPU (reads are independent: no collective)."""
import argparse
import os
import sys
import time

import numpy as np

MAX_SLEEP = 0.01
EVENTS_COLUMNS = ("read_id", "start", "length", "mean", "stdv", "norm_scale", "norm_shift", "norm_mean", "win_mean",
                  "win_stdv", "win_mask")


def get_parser(conf):
    from . import index_params as IP
    D = IP.DEFAULTS
    fmt = argparse.ArgumentDefaultsHelpFormatter
    parser = argparse.ArgumentParser(prog="uncalled_b200", description="Rapidly maps raw nanopore signal to DNA references",
                                     formatter_class=fmt)
    sp = parser.add_subparsers(dest="subcmd")
    p = sp.add_parser("index", help="Builds the UNCALLED index of a FASTA reference", formatter_class=fmt)
    p.add_argument("fasta_filename", type=str, help="FASTA file to index")
    p.add_argument("-o", "--bwa-prefix", type=str, default=None, help="Index output prefix. Will use input fasta filename by default")
    p.add_argument("-s", "--max-sample-dist", type=int, default=D["max_sample_dist"], help="Maximum average sampling distance between reference alignments.")
    p.add_argument("--min-samples", type=int, default=D["min_samples"], help="Minimum number of alignments to produce")
    p.add_argument("--max-samples", type=int, default=D["max_samples"], help="Maximum number of alignments to produce")
    p.add_argument("-k", "--kmer-len", type=int, default=D["kmer_len"], help="Model k-mer length")
    p.add_argument("-1", "--matchpr1", type=float, default=D["matchpr1"], help="Minimum event match probability")
    p.add_argument("-2", "--matchpr2", type=float, default=D["matchpr2"], help="Maximum event match probability")
    p.add_argument("-f", "--pathlen-percentile", type=float, default=D["pathlen_percentile"], help="")
    p.add_argument("-m", "--max-replen", type=int, default=D["max_replen"], help="")
    p.add_argument("--probs", type=str, default=None, help="Find parameters with specified target probabilites (comma separated)")
    p.add_argument("--speeds", type=str, default=None, help="Find parameters with specified speed coefficents (comma separated)")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("map", help="Map fast5 files to a DNA reference", formatter_class=fmt)
    p.add_argument("bwa_prefix", type=str, help="BWA prefix to mapping to. Must be processed by \"uncalled index\".")
    p.add_argument("-p", "--idx-preset", type=str, default=conf.idx_preset, help="Mapping mode")
    p.add_argument("fast5s", nargs="+", type=str, help="Reads to map. Can be a directory which will be recursively searched "
                   "for all files with the \".fast5\" extension, a text file containing one fast5 filename per line, or a "
                   "comma-separated list of fast5 file names.")
    p.add_argument("-r", "--recursive", action="store_true")
    p.add_argument("-l", "--read-list", type=str, default=None, help=type(conf).read_list.__doc__)
    p.add_argument("-n", "--max-reads", type=int, default=None, help=type(conf).max_reads.__doc__)
    p.add_argument("-t", "--threads", type=int, default=conf.threads, help="Number of host threads (fast5 decoding; the mapping runs on the GPU)")
    p.add_argument("--num-channels", type=int, default=conf.num_channels, help="Number of channels used in sequencing.")
    p.add_argument("-e", "--max-events", type=int, default=conf.max_events, help="Will give up on a read after this many events have been processed")
    p.add_argument("-c", "--max-chunks", type=int, default=conf.max_chunks, help="Will give up on a read after this many chunks have been processed.")
    p.add_argument("--chunk-time", type=float, default=1, required=False, help="Length of chunks in seconds")
    p.add_argument("--device", type=int, default=conf.device, help="CUDA device")
    p.add_argument("--batch-reads", type=int, default=conf.batch_reads, help="Reads per GPU batch")
    p.add_argument("--ordered", action="store_const", const=1, default=conf.ordered, help=type(conf).ordered.__doc__)
    p.add_argument("--exact-ties", action="store_const", const=1, default=conf.exact_ties, help=type(conf).exact_ties.__doc__)

    p = sp.add_parser("map-ord", help="Map fast5 files as UNCALLED would have in real time: every channel's reads replayed "
                      "in the order they were sequenced, chunk by chunk, through the streaming mapper", formatter_class=fmt)
    p.add_argument("bwa_prefix", type=str, help="BWA prefix to mapping to. Must be processed by \"uncalled index\".")
    p.add_argument("-p", "--idx-preset", type=str, default=conf.idx_preset, help="Mapping mode")
    p.add_argument("fast5s", nargs="+", type=str, help="Reads to map. Can be a directory which will be recursively searched "
                   "for all files with the \".fast5\" extension, a text file containing one fast5 filename per line, or a "
                   "comma-separated list of fast5 file names.")
    p.add_argument("-r", "--recursive", action="store_true")
    p.add_argument("-l", "--read-list", type=str, default=None, help=type(conf).read_list.__doc__)
    p.add_argument("-n", "--max-reads", type=int, default=None, help=type(conf).max_reads.__doc__)
    p.add_argument("-t", "--threads", type=int, default=conf.threads, help="Number of host threads (fast5 decoding; the mapping runs on the GPU)")
    p.add_argument("--num-channels", type=int, default=conf.num_channels, help="Number of channels used in sequencing.")
    p.add_argument("-e", "--max-events", type=int, default=conf.max_events, help="Will give up on a read after this many events have been processed")
    p.add_argument("-c", "--max-chunks", type=int, default=conf.max_chunks, help="Will give up on a read after this many chunks have been processed.")
    p.add_argument("--chunk-time", type=float, default=1, required=False, help="Length of chunks in seconds")
    p.add_argument("--min-active-reads", type=int, default=conf.min_active_reads, help=type(conf).min_active_reads.__doc__)
    p.add_argument("--exact-ties", action="store_const", const=1, default=conf.exact_ties, help=type(conf).exact_ties.__doc__)
    p.add_argument("--device", type=int, default=conf.device, help="CUDA device")

    p = sp.add_parser("sim", help="Simulate real-time targeted sequencing (read until) from a control run and an "
                      "UNCALLED run", formatter_class=fmt)
    p.add_argument("bwa_prefix", type=str, help="BWA prefix to mapping to. Must be processed by \"uncalled index\".")
    p.add_argument("-p", "--idx-preset", type=str, default=conf.idx_preset, help="Mapping mode")
    p.add_argument("fast5s", nargs="+", type=str, help="Reads of the control run. Can be a directory which will be "
                   "recursively searched for all files with the \".fast5\" extension, a text file containing one fast5 "
                   "filename per line, or a comma-separated list of fast5 file names.")
    p.add_argument("-r", "--recursive", action="store_true")
    p.add_argument("--ctl-seqsum", type=str, required=True, help=type(conf).ctl_seqsum.__doc__)
    p.add_argument("--unc-seqsum", type=str, required=True, help=type(conf).unc_seqsum.__doc__)
    p.add_argument("--unc-paf", type=str, required=True, help=type(conf).unc_paf.__doc__)
    p.add_argument("--sim-speed", type=float, default=conf.sim_speed, help=type(conf).sim_speed.__doc__)
    p.add_argument("-t", "--threads", type=int, default=conf.threads, help="Number of host threads (fast5 decoding; the mapping runs on the GPU)")
    p.add_argument("--num-channels", type=int, default=conf.num_channels, help="Number of channels used in sequencing.")
    p.add_argument("-e", "--max-events", type=int, default=conf.max_events, help="Will give up on a read after this many events have been processed")
    p.add_argument("-c", "--max-chunks", type=int, default=conf.max_chunks, help="Will give up on a read after this many chunks have been processed.")
    p.add_argument("--chunk-time", type=float, default=1, required=False, help="Length of chunks in seconds")
    p.add_argument("--exact-ties", action="store_const", const=1, default=conf.exact_ties, help=type(conf).exact_ties.__doc__)
    from .api import RealtimePool as RP
    modes = p.add_mutually_exclusive_group(required=True)          # uncalled/args.py:161-188
    modes.add_argument("-D", "--deplete", action="store_const", const=RP.DEPLETE, dest="realtime_mode",
                       help="Will eject reads that align to index")
    modes.add_argument("-E", "--enrich", action="store_const", const=RP.ENRICH, dest="realtime_mode",
                       help="Will eject reads that don't align to index")
    active = p.add_mutually_exclusive_group()
    active.add_argument("--full", action="store_const", const=RP.FULL, dest="active_chs", help="Will monitor all pores if set (default)")
    active.add_argument("--even", action="store_const", const=RP.EVEN, dest="active_chs", help="Will only monitor even pores if set")
    active.add_argument("--odd", action="store_const", const=RP.ODD, dest="active_chs", help="Will only monitor odd pores if set")
    p.add_argument("--device", type=int, default=conf.device, help="CUDA device")

    p = sp.add_parser("mask-internal", help="Iteratively masks the most frequent k-mer of a FASTA reference with N "
                      "(masking/mask_internal.sh)", formatter_class=fmt)
    p.add_argument("reference", type=str, help="fasta file of the reference to mask")
    p.add_argument("k", type=int, help="k-mer length (1 to 13)")
    p.add_argument("iters", type=int, help="number of masking iterations to run")
    p.add_argument("out_prefix", type=str, help="output prefix: writes <out_prefix>mask<iters>.fa")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("mask-external", help="Masks the windows of a target reference that occur more than min_copy "
                      "times in a full reference, on either strand (masking/mask_external.sh)", formatter_class=fmt)
    p.add_argument("full_reference", type=str, help="fasta file of the full reference (e.g. the whole genome)")
    p.add_argument("target", type=str, help="fasta file of the target reference to mask")
    p.add_argument("min_len", type=int, help="window length (2 to 64)")
    p.add_argument("min_copy", type=int, help="windows with more than this many copies are masked")
    p.add_argument("out_prefix", type=str, help="output prefix: writes <out_prefix>masked<min_copy>.fa and "
                   "<out_prefix>reps_m<min_copy>.bed")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("dtw", help="Align reads to known reference spans at the signal level (DTW of the read's "
                      "normalised event means against the span's k-mers)", formatter_class=fmt)
    p.add_argument("bwa_prefix", type=str, help="BWA prefix of the reference (only the .pac and .ann are read)")
    p.add_argument("fast5s", nargs="+", type=str, help="Reads to align. Can be a directory which will be recursively "
                   "searched for all files with the \".fast5\" extension, a text file containing one fast5 filename per "
                   "line, or a comma-separated list of fast5 file names.")
    p.add_argument("--queries", required=True, type=str, help="One query per line: rd_name rd_st rd_en rf_name rf_st "
                   "rf_en strand (samples [rd_st, rd_en) of the read, 0 0 = all of it; bases [rf_st, rf_en) of the contig)")
    p.add_argument("--path-prefix", type=str, default="", help="Also write each read's DTW path to <prefix><read_id>.txt")
    p.add_argument("--band", type=int, default=0, help="Align within this many rows (k-mers) of the diagonal instead of "
                   "the whole matrix (0: the whole matrix, and reads over 50 000 kept means are skipped)")
    p.add_argument("-r", "--recursive", action="store_true", help="Recursively search 'fast5s' for fast5 files")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("events", help="Write every event of every read with the mapper's normalisation and stall mask "
                      "(the reference's DEBUG_EVENTS columns) as one TSV on stdout", formatter_class=fmt,
                      description="One row per event, reads in input order, columns: " + " ".join(EVENTS_COLUMNS) + ". "
                      "Floats are printed with %%.9g so that they read back to the same float32 (the reference's "
                      "debug file prints 6 significant digits).  win_mean and win_stdv are nan for the last events of "
                      "a read, which never reach the middle of the profiler's window.  The whole signal is used.")
    p.add_argument("fast5s", nargs="+", type=str, help="Reads. Can be a directory which will be searched for all files with "
                   "the \".fast5\" extension, a text file containing one fast5 filename per line, or a fast5 file.")
    p.add_argument("-r", "--recursive", action="store_true", help="Recursively search 'fast5s' for fast5 files")
    p.add_argument("-l", "--read-list", type=str, default=None, help="Only write reads listed in this file")
    p.add_argument("-n", "--max-reads", type=int, default=None, help="Maximum number of reads to write")
    p.add_argument("--model", type=str, default=None, help="Pore model table (1024 x {mean, stdv} float32, template "
                   "k-mer order); default: the built-in r9.4 model")
    p.add_argument("--batch-reads", type=int, default=256, help="Reads per GPU batch")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("find-repeats", help="Report how long the sequence at each reference position stays repeated in the "
                      "reference and its reverse complement (src/find_repeats.cpp)", formatter_class=fmt,
                      description="One line per position whose repeat length L is at least min_k: L, contig, p, p + L and "
                      "the contig's bases [p, p + L) (N inside .amb holes).  L is the number of FM-index steps after "
                      "which the bases from p are unique or the contig ends.  Positions inside .amb holes are not reported.")
    p.add_argument("bwa_prefix", type=str, help="BWA prefix of the reference (.bwt, .sa, .pac, .ann and .amb are read)")
    p.add_argument("min_k", type=int, help="report positions with a repeat length of at least this (0: every position)")
    p.add_argument("--bed", action="store_true", help="write the merged intervals [p, p + L) of the reported positions as "
                   "BED instead")
    p.add_argument("--device", type=int, default=0, help="CUDA device")

    p = sp.add_parser("pafstats",help="Computes speed and accuracy of UNCALLED mappings.", formatter_class=fmt)
    p.add_argument("infile", type=str, help="PAF file output by UNCALLED")          # uncalled/pafstats.py:165-169
    p.add_argument("-n", "--max-reads", required=False, type=int, default=None, help="Will only look at first n reads if specified")
    p.add_argument("-r", "--ref-paf", required=False, type=str, default=None, help="Reference PAF file. Will output percent true/false "
                   "positives/negatives with respect to reference. Reads not mapped in reference PAF will be classified as NA.")
    return parser


def fast5_path(fname):
    if fname.startswith("#") or not fname.endswith("fast5"):
        return None
    path = os.path.abspath(fname)
    if not os.path.isfile(path):
        sys.stderr.write("Warning: \"%s\" is not a fast5 file.\n" % fname)
        return None
    return path


def load_fast5s(fast5s, recursive):
    """scripts/uncalled:88-118: directories (optionally recursive), .fast5 files, or text files of file names."""
    for path in fast5s:
        path = path.strip()
        if not os.path.exists(path):
            sys.stderr.write("Error: \"%s\" does not exist\n" % path)
            sys.exit(1)
        if os.path.isdir(path) and recursive:
            for root, _, files in os.walk(path):
                for fname in files:
                    yield fast5_path(os.path.join(root, fname))
        elif os.path.isdir(path):
            for fname in os.listdir(path):
                yield fast5_path(os.path.join(path, fname))
        elif path.endswith(".fast5"):
            yield fast5_path(path)
        else:
            with open(path) as infile:
                for line in infile:
                    yield fast5_path(line.strip())


def assert_exists(fname):
    if not os.path.exists(fname):
        sys.stderr.write("Error: '%s' does not exist\n" % fname)
        sys.exit(1)


def index_cmd(args):
    from . import _native as N
    from . import index as UI
    N.check(N.lib().unc_init(args.device))
    opts = {k: getattr(args, k) for k in ("max_sample_dist", "min_samples", "max_samples", "kmer_len", "matchpr1", "matchpr2",
                                          "pathlen_percentile", "max_replen")}
    UI.index_cmd(args.fasta_filename, args.bwa_prefix, probs=args.probs, speeds=args.speeds, **opts)


def map_cmd(conf, args, out=None):
    from .api import MapPool
    assert_exists(conf.bwa_prefix + ".bwt")
    assert_exists(conf.bwa_prefix + ".uncl")
    if len(conf.read_list) > 0:
        assert_exists(conf.read_list)
    # one process per GPU (torchrun / mpirun): rank r maps the files i with i mod WORLD_SIZE == r on GPU LOCAL_RANK
    world, rank = int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("RANK", "0"))
    if world > 1:
        conf.device = int(os.environ.get("LOCAL_RANK", rank))
    mapper = MapPool(conf)
    sys.stderr.write("Loading fast5s\n")
    from .shard import local_files
    files = [f for f in load_fast5s(args.fast5s, args.recursive) if f is not None]
    for fast5 in local_files(files, world, rank):
        mapper.add_fast5(fast5)
    sys.stderr.write("Mapping\n")
    sys.stderr.flush()
    try:
        while mapper.running():
            t0 = time.time()
            for p in mapper.update():
                p.print_paf(out)
            dt = time.time() - t0
            if dt < MAX_SLEEP:
                time.sleep(MAX_SLEEP - dt)
    except KeyboardInterrupt:
        pass
    sys.stderr.write("Finishing\n")
    mapper.stop()


def map_ord_cmd(conf, args, out=None, backend=None, index=None):
    """uncalled_map_ord (reference src/uncalled_map_ord.cpp): every read is loaded up front, then the channels are replayed
    on the device; PAF goes to `out` (stdout), progress to stderr.  A missing index file or read list, or a read on a
    channel above --num-channels, ends the command with status 1 before the GPU is touched."""
    from .api import MapPoolOrd
    if backend is None:
        assert_exists(conf.bwa_prefix + ".bwt")
        assert_exists(conf.bwa_prefix + ".uncl")
    if len(conf.read_list) > 0:
        assert_exists(conf.read_list)
    pool = MapPoolOrd(conf, backend=backend, index=index)
    for fast5 in load_fast5s(args.fast5s, args.recursive):
        if fast5 is not None:
            pool.add_fast5(fast5)
    sys.stderr.write("Loading fast5s\n")
    try:
        pool.load_fast5s()
    except ValueError as e:
        sys.stderr.write("Error: %s\n" % e)
        sys.exit(1)
    sys.stderr.write("Mapping\n")
    sys.stderr.flush()
    try:
        while pool.running():
            for p in pool.update():
                p.print_paf(out)
    except KeyboardInterrupt:
        pass
    sys.stderr.write("Finishing\n")
    pool.stop()


def sim_cmd(conf, args, out=None):
    """scripts/uncalled:169-300 with `sim`: the pattern and the control reads are loaded, then the decision loop runs
    until every simulated channel has run out.  Bad input ends the command with status 1 before the GPU is touched."""
    from .sim import SimError, run_sim
    assert_exists(conf.bwa_prefix + ".bwt")
    assert_exists(conf.bwa_prefix + ".uncl")
    files = [f for f in load_fast5s(args.fast5s, args.recursive) if f is not None]
    try:
        run_sim(conf, files, out)
    except SimError as e:
        sys.stderr.write("Error: %s\n" % e)
        sys.exit(1)
    sys.stderr.write("Finished\n")


def dtw_cmd(args, out=None):
    """src/dtw_test.cpp: the reads named in the query file, in the order the fast5 files hand them out, aligned on the GPU.
    stdout: read_id, mean score, seconds.  A bad query file ends the command with status 1 before the GPU is touched."""
    from concurrent.futures import ThreadPoolExecutor
    from . import _native as N
    from .dtw import DtwAligner, QueryError, format_path, host_skip, load_queries
    from .fast5 import Fast5File
    out = out or sys.stdout
    for ext in (".pac", ".ann"):
        assert_exists(args.bwa_prefix + ext)
    assert_exists(args.queries)
    if not 0 <= args.band < 1 << 32:
        sys.stderr.write("Error: --band must be 0 (the whole matrix) or a half-width below 2^32\n")
        sys.exit(1)
    aligner = DtwAligner(args.bwa_prefix, band=args.band)
    try:
        queries = load_queries(args.queries, aligner)
    except QueryError as e:
        sys.stderr.write("Error: %s\n" % e)
        sys.exit(1)
    files = [f for f in load_fast5s(args.fast5s, args.recursive) if f is not None]

    def batches(max_reads=64, max_samples=1 << 25):
        """the queried reads, decoded file by file (Fast5Reader::add_read filter), in batches of one signal type"""
        batch, n = [], 0
        for path in files:
            with Fast5File(path) as f:
                for i in range(f.n_reads):
                    if f.info(i).read_id not in queries:
                        continue
                    r = f.load(i, 1)[0]
                    if batch and (len(batch) >= max_reads or n + len(r.signal) > max_samples):
                        yield batch
                        batch, n = [], 0
                    batch.append(r)
                    n += len(r.signal)
        if batch:
            yield batch

    gpu_ready = False
    with ThreadPoolExecutor(max_workers=1) as ex:     # the next batch is decoded while the GPU aligns this one
        it = batches()
        fut = ex.submit(next, it, None)
        while True:
            batch = fut.result()
            if batch is None:
                break
            fut = ex.submit(next, it, None)
            t0 = time.time()
            qs = [(r.read_id, r.signal, r.calibration) + queries[r.read_id] for r in batch]
            if not gpu_ready and any(host_skip(aligner, len(q[1]), *q[3:8]) is None for q in qs):
                N.check(N.lib().unc_init(args.device))
                gpu_ready = True
            res = aligner.align(qs, paths=bool(args.path_prefix))
            secs = (time.time() - t0) / len(res)
            for a in res:
                if a.skip is not None:
                    sys.stderr.write(a.skip_message() + "\n")
                    continue
                if args.path_prefix:
                    with open(args.path_prefix + a.read_id + ".txt", "w") as pf:
                        pf.write(format_path(a))
                out.write("%s\t%g\t%g\n" % (a.read_id, a.mean_score, secs))
            out.flush()


def events_cmd(args, out=None):
    """`events`: every event of the selected reads (uncalled_b200.signal) as TSV on `out` (stdout).  The next batch is
    decoded on a host thread while the GPU processes this one.  A bad argument or a missing file ends the command with
    status 1 before the GPU is touched."""
    from concurrent.futures import ThreadPoolExecutor
    from .fast5 import Fast5File
    from .signal import SignalProcessor
    out = out or sys.stdout
    if args.max_reads is not None and args.max_reads < 0:
        sys.stderr.write("Error: --max-reads must not be negative\n")
        sys.exit(1)
    if args.batch_reads < 1:
        sys.stderr.write("Error: --batch-reads must be at least 1\n")
        sys.exit(1)
    if args.device < 0:
        sys.stderr.write("Error: --device must not be negative\n")
        sys.exit(1)
    if args.model is not None:
        assert_exists(args.model)
        if os.path.getsize(args.model) != 1024 * 2 * 4:
            sys.stderr.write("Error: '%s' is not a pore model table of 1024 (mean, stdv) float32 pairs\n" % args.model)
            sys.exit(1)
    ids = None
    if args.read_list:
        assert_exists(args.read_list)
        ids = set(l.strip() for l in open(args.read_list) if l.strip())
    files = [f for f in load_fast5s(args.fast5s, args.recursive) if f is not None]
    cap = args.max_reads or 0

    def batches():
        """the selected reads, whole signals, in file order, batch_reads at a time"""
        batch, n = [], 0
        for path in files:
            with Fast5File(path) as f:
                for i in range(f.n_reads):
                    if cap and n >= cap:
                        break
                    if ids is not None and f.info(i).read_id not in ids:
                        continue
                    batch.append(f.load(i, 1)[0])
                    n += 1
                    if len(batch) >= args.batch_reads:
                        yield batch
                        batch = []
            if cap and n >= cap:
                break
        if batch:
            yield batch

    out.write("\t".join(EVENTS_COLUMNS) + "\n")
    proc = None
    with ThreadPoolExecutor(max_workers=1) as ex:
        it = batches()
        fut = ex.submit(next, it, None)
        while True:
            batch = fut.result()
            if batch is None:
                break
            fut = ex.submit(next, it, None)
            if proc is None:
                proc = SignalProcessor(model_path=args.model, device=args.device)
            res = proc.run([r.signal for r in batch], [r.calibration for r in batch])
            out.write(format_events([r.read_id for r in batch], res))
            out.flush()


def find_repeats_cmd(args, out=None):
    """`find-repeats`: the reported positions' lines, or their BED with --bed, on `out` (stdout).  A negative min_k or a
    missing or inconsistent index ends the command with status 1 before the GPU is touched."""
    from .repeats import IndexFileError, RepeatFinder, write_bed, write_lines
    out = out or sys.stdout
    if args.min_k < 0:
        sys.stderr.write("Error: min_k must be 0 or more\n")
        sys.exit(1)
    try:
        finder = RepeatFinder(args.bwa_prefix, device=args.device)
    except IndexFileError as e:
        sys.stderr.write("Error: %s\n" % e)
        sys.exit(1)
    try:
        (write_bed if args.bed else write_lines)(finder, args.min_k, out)
    finally:
        finder.close()
    out.flush()


def _g9(a):
    """%.9g of every value of a float32 array (reads back to the same float32), as a list of strings"""
    return ["%.9g" % x for x in np.asarray(a, np.float64).tolist()]


def format_events(read_ids, res):
    """TSV rows of an EventBatch (EVENTS_COLUMNS without the header), formatted column by column"""
    ev = res.events
    if ev is None or len(ev) == 0:
        return ""
    n = res.reads["n_events"].astype(np.int64)
    per_read = lambda v: np.repeat(np.asarray(v, dtype=object), n).tolist()   # noqa: E731
    cols = [per_read(list(read_ids)), ev["start"].astype(str).tolist(), _g9(ev["length"]), _g9(ev["mean"]),
            _g9(ev["stdv"]), per_read(_g9(res.reads["norm_scale"])), per_read(_g9(res.reads["norm_shift"])),
            _g9(ev["norm_mean"]), _g9(ev["win_mean"]), _g9(ev["win_stdv"]), ev["win_mask"].astype(str).tolist()]
    return "".join("\t".join(row) + "\n" for row in zip(*cols))


def load_conf(argv):
    """uncalled/args.py:288-302: every parsed option whose name is a Conf attribute is set on the Conf."""
    from .api import Conf
    conf = Conf()
    parser = get_parser(conf)
    args = parser.parse_args(argv)
    for a, v in vars(args).items():
        if v is not None and not a.startswith("_") and hasattr(conf, a):
            setattr(conf, a, v)
    return parser, conf, args


def main(argv=None):
    parser, conf, args = load_conf(sys.argv[1:] if argv is None else argv)
    if args.subcmd == "index":
        index_cmd(args)
    elif args.subcmd == "map":
        map_cmd(conf, args)
    elif args.subcmd == "map-ord":
        map_ord_cmd(conf, args)
    elif args.subcmd == "sim":
        sim_cmd(conf, args)
    elif args.subcmd == "mask-internal":
        from . import _native as N
        from .mask import mask_internal
        assert_exists(args.reference)
        N.check(N.lib().unc_init(args.device))
        done = mask_internal(args.reference, args.k, args.iters, args.out_prefix)
        if len(done) < args.iters:
            sys.stderr.write("No k-mer left to mask after %d iterations\n" % len(done))
    elif args.subcmd == "mask-external":
        from . import _native as N
        from .mask import mask_external
        assert_exists(args.full_reference)
        assert_exists(args.target)
        N.check(N.lib().unc_init(args.device))
        masked, _ = mask_external(args.full_reference, args.target, args.min_len, args.min_copy, args.out_prefix)
        sys.stdout.write("Masked %d basepairs\n" % masked)
    elif args.subcmd == "dtw":
        dtw_cmd(args)
    elif args.subcmd == "events":
        events_cmd(args)
    elif args.subcmd == "find-repeats":
        find_repeats_cmd(args)
    elif args.subcmd == "pafstats":
        from . import pafstats
        pafstats.run(args.infile, args.ref_paf, args.max_reads)
    else:
        parser.print_help()
    return 0
