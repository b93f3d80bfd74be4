#!/bin/bash
# k_lsd_grow_ordered time of one launch at several batch sizes (CUDA events inside the library); every run has its own hard limit
for B in ${BATCHES:-1 8 64 512 4224}; do echo "B=$B"; B=$B timeout -k 5 100 python tools/bench_grow.py pl-slam_b200/libplslam_b200.so 2>&1 | tail -2; done
