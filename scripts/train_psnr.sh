#!/bin/bash
# PSNR of the UNMODIFIED trainer (ExpRunner::Train -> TestImages, src/ExpRunner.cpp:65-186,322-391) on the reference's ngp_fox
# example, twice on the same box with the same config and seed (main.cpp: torch::manual_seed(2022)):
#   reference arm   oracle/_ref/ref_driver      --train   (Totoro97/f2-nerf + tiny-cuda-nn, nothing replaced)
#   b200 arm        oracle/_ref/ref_driver_b200 --train   (same program, Renderer::Render = f2nerf_b200/shim/B200Renderer.cpp)
# usage: scripts/train_psnr.sh [end_iter=20000]      -> gpurun_out/train_psnr.json + the two logs
# ARMS="ref" or ARMS="b200" trains one arm only.  Each arm leaves its experiment directory (checkpoints/latest, test_images)
# in /tmp/f2b_train_<arm> and its config in /tmp/f2b_train_<arm>.yaml; scripts/eval_trained.py evaluates them on the device.
set -u
cd "$(dirname "$0")/.."
END=${1:-20000}
mkdir -p gpurun_out
for arm in ${ARMS:-ref b200}; do
  exp=/tmp/f2b_train_$arm
  rm -rf $exp
  sed -e "s|^base_exp_dir: .*|base_exp_dir: $exp|" -e "s|^  end_iter: .*|  end_iter: $END|" oracle/ref_config_ngp_fox.yaml > /tmp/f2b_train_$arm.yaml
  bin=oracle/_ref/ref_driver; [ $arm = b200 ] && bin=oracle/_ref/ref_driver_b200
  start=$(date +%s)
  timeout 3000 $bin --train /tmp/f2b_train_$arm.yaml > gpurun_out/train_$arm.log 2>&1
  echo "rc=$? wall_s=$(( $(date +%s) - start ))" >> gpurun_out/train_$arm.log
  cp $exp/test_images/info.yaml gpurun_out/train_${arm}_info.yaml 2>/dev/null
  cp $exp/train_info.txt gpurun_out/train_${arm}_seconds.txt 2>/dev/null
done
python - "$END" <<'PY'
import json, re, sys
out = {"end_iter": int(sys.argv[1]), "config": "oracle/ref_config_ngp_fox.yaml (confs/wanjinyou.yaml flattened), ngp_fox factor 2, 7 test images"}
for arm in ("ref", "b200"):
    try:
        log = open(f"gpurun_out/train_{arm}.log", errors="ignore").read()
    except FileNotFoundError:                                   # an arm left out through ARMS
        continue
    it = re.findall(r"Iter:\s+(\d+) PSNR: ([\d.]+) NRays:\s+(\d+) OctSamples: ([\d.]+) Samples: ([\d.]+) MeaningfulSamples: ([\d.]+) IPS: ([\d.]+)", log)
    mean = re.findall(r"Mean psnr: ([\d.]+)", log)
    rc = re.findall(r"rc=(\d+) wall_s=([\d.]+)", log)
    try:
        secs = float(open(f"gpurun_out/train_{arm}_seconds.txt").read().split()[0])
    except Exception:
        secs = None
    pick = [r for r in it if int(r[0]) % max(int(sys.argv[1]) // 10, 50) == 0]
    out[arm] = {"rc": int(rc[-1][0]) if rc else None, "wall_s": float(rc[-1][1]) if rc else None, "train_seconds": secs,
                "test_mean_psnr": float(mean[-1]) if mean else None, "nan_skips": log.count("Nan!"),
                "train_psnr_smooth": [{"iter": int(r[0]), "psnr": float(r[1]), "n_rays": int(r[2]), "samples": float(r[4]),
                                       "meaningful": float(r[5]), "ips": float(r[6])} for r in pick]}
json.dump(out, open("gpurun_out/train_psnr.json", "w"), indent=1)
print(json.dumps({k: (v if not isinstance(v, dict) else {kk: v[kk] for kk in ("rc", "wall_s", "train_seconds", "test_mean_psnr", "nan_skips")}) for k, v in out.items()}))
PY
