#!/bin/bash
# the final build's C++ host through the unmodified trainer, full 20 000-iteration schedule (drop-in arm only; the reference arm's
# 20 k run of this round is profiles/r02e_train_psnr_20k.json)
cd "$(dirname "$0")/.."
O=gpurun_out; mkdir -p $O; TAG=${TAG:-r02o}
sed -e "s|^base_exp_dir: .*|base_exp_dir: /tmp/f2b_train_final20k|" oracle/ref_config_ngp_fox.yaml > /tmp/f2b_final20k.yaml
rm -rf /tmp/f2b_train_final20k
start=$(date +%s)
F2B_SHIM_PROFILE=1 timeout 1500 oracle/_ref/ref_driver_b200 --train /tmp/f2b_final20k.yaml > $O/${TAG}_train_b200.log 2>&1; echo "--- b200 trainer rc=$? wall_s=$(( $(date +%s) - start ))"
grep -E "Iter: +(5000|10000|15000|20000) |^[0-9]+: |Mean psnr|f2b_shim_profile|Nan" $O/${TAG}_train_b200.log | cut -c1-200; cat /tmp/f2b_train_final20k/train_info.txt
