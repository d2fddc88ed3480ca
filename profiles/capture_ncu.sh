#!/bin/bash
# One `ncu --set full` capture per hot kernel (cold caches, clocks not locked), reports into gpurun_out/<tag>_<name>.ncu-rep.
#   bash profiles/capture_ncu.sh <tag> [names...]   names: convh convh_glu convh_acc wgradh conv conv_glu conv_acc wgrad scores_train bn_bwd bn_fwd
tag=$1; shift
names=${@:-conv conv_glu conv_acc wgrad scores_train bn_bwd bn_fwd}
for n in $names; do
  case $n in
    convh|convh_glu|convh_acc) k=conv_hp_kernel; c=1;;
    wgradh) k=wgrad_hp_kernel; c=1;;
    conv|conv_glu|conv_acc) k=conv_pp_kernel; c=1;;
    wgrad) k=wgrad_pp_kernel; c=1;;
    scores_train) k=clip_scores_kernel; c=1;;
    bn_bwd) k=epi_bwd; c=2;;
    bn_fwd) k=epi_fwd; c=1;;
  esac
  s=$((3 * c))
  timeout 300 ncu --set full --clock-control none --import-source on -k regex:$k -s $s -c $c -f -o gpurun_out/${tag}_${n} \
      python profiles/profile_kernels.py $n > gpurun_out/${tag}_${n}.log 2>&1
  echo "$n rc=$?"
done
