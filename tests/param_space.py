"""The mapping cases of tests/golden/synth_params (make_golden_params.sh): the synth_small reads at index shapes other than
(17, 7) and at mapping knobs the other goldens leave at their defaults.  name -> (k, w, single_end, preset, parameter overrides)."""

PARAM_CASES = {
    "mfl70": (19, 10, False, "", {}),                                      # --min-frag-length 70
    "mfl70_e15": (19, 10, False, "", dict(error_threshold=15)),
    "mfl100_q0": (23, 11, False, "", dict(mapq_threshold=0)),              # --min-frag-length 100: k > 22
    "mfl100_chip": (23, 11, False, "chip", {}),
    "mfl100_se_q0": (23, 11, True, "", dict(mapq_threshold=0)),
    "k28w20": (28, 20, False, "", {}),                                     # the largest k the library accepts
    "k16w5_q0": (16, 5, False, "", dict(mapq_threshold=0)),                # even k: strand-symmetric k-mers
    "e15q0": (17, 7, False, "", dict(error_threshold=15, mapq_threshold=0)),   # the widest band
    "e7q0": (17, 7, False, "", dict(error_threshold=7, mapq_threshold=0)),     # the last error threshold with 8 lanes
    "e1q0": (17, 7, False, "", dict(error_threshold=1, mapq_threshold=0)),     # the narrowest band
    "n8q0": (17, 7, False, "", dict(max_num_best_mappings=8, mapq_threshold=0)),
    "s1q0": (17, 7, False, "", dict(min_num_seeds=1, mapq_threshold=0)),
    "s4": (17, 7, False, "", dict(min_num_seeds=4)),
    "f20_200q0": (17, 7, False, "", dict(max_seed_freq0=20, max_seed_freq1=200, mapq_threshold=0)),
    "drop30q0": (17, 7, False, "", dict(drop_repetitive_reads=30, mapq_threshold=0)),
    "minlen45q0": (17, 7, False, "", dict(min_read_length=45, mapq_threshold=0)),
    "se_e15n8q0": (17, 7, True, "", dict(error_threshold=15, max_num_best_mappings=8, mapq_threshold=0)),
}

SHAPES = sorted({(k, w) for k, w, _, _, _ in PARAM_CASES.values()})
