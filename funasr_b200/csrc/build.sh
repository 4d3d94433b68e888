#!/bin/bash
# Builds libfunasr_b200.so in-tree for sm_90a (cross-compiles without a GPU).
set -e
cd "$(dirname "$0")"
NVCC=${NVCC:-/usr/local/cuda/bin/nvcc}
FLAGS="-gencode arch=compute_90a,code=sm_90a -O3 -lineinfo -std=c++17 -Xcompiler -fPIC -Xptxas -v --expt-relaxed-constexpr"
mkdir -p ../_build
# objects built with other flags (another architecture) are stale even when newer than their sources
if [ "$(cat ../_build/flags 2>/dev/null)" != "$FLAGS" ]; then rm -f ../_build/*.o; echo "$FLAGS" > ../_build/flags; fi
objs=""
pids=""
for f in fbank layernorm gemm_f32 gemm_tc attention_tc attention_f32 fsmn cif decode_ops model handle_core offline_asr offline_vad offline_spk offline_long offline_pool offline_punc offline_align lstm hotword resample vad campplus spk_cluster; do
  if [ ! -f ../_build/$f.o ] || [ $f.cu -nt ../_build/$f.o ] || [ common.cuh -nt ../_build/$f.o ] || [ kernels.h -nt ../_build/$f.o ] || [ handle.h -nt ../_build/$f.o ] || [ request_pool.h -nt ../_build/$f.o ] || [ tc_common.cuh -nt ../_build/$f.o ] || [ ../../include/funasr_b200.h -nt ../_build/$f.o ] || [ punc_text.h -nt ../_build/$f.o ]; then
    ( $NVCC $FLAGS -c $f.cu -o ../_build/$f.o 2> ../_build/$f.ptxas.log || { cat ../_build/$f.ptxas.log; rm -f ../_build/$f.o; exit 1; } ) &
    pids="$pids $!"
  fi
  objs="$objs ../_build/$f.o"
done
# host-only C++: the FunOffline* shim with the reference runtime's C++ signatures (include/funasrruntime_b200.h)
if [ ! -f ../_build/runtime_shim.o ] || [ runtime_shim.cpp -nt ../_build/runtime_shim.o ] || [ ../../include/funasrruntime_b200.h -nt ../_build/runtime_shim.o ] || [ ../../include/funasr_b200.h -nt ../_build/runtime_shim.o ]; then
  ( g++ -O2 -std=c++17 -fPIC -c runtime_shim.cpp -o ../_build/runtime_shim.o 2> ../_build/runtime_shim.log || { cat ../_build/runtime_shim.log; rm -f ../_build/runtime_shim.o; exit 1; } ) &
  pids="$pids $!"
fi
objs="$objs ../_build/runtime_shim.o"
# host-only C++: the FSMN-VAD end-point detector (fa_vad_detect_segments)
if [ ! -f ../_build/vad_detector.o ] || [ vad_detector.cpp -nt ../_build/vad_detector.o ] || [ ../../include/funasr_b200.h -nt ../_build/vad_detector.o ]; then
  ( g++ -O2 -std=c++17 -fPIC -ffp-contract=off -c vad_detector.cpp -o ../_build/vad_detector.o 2> ../_build/vad_detector.log || { cat ../_build/vad_detector.log; rm -f ../_build/vad_detector.o; exit 1; } ) &
  pids="$pids $!"
fi
objs="$objs ../_build/vad_detector.o"
if [ ! -f ../_build/host_ops.o ] || [ host_ops.cpp -nt ../_build/host_ops.o ] || [ ../../include/funasr_b200.h -nt ../_build/host_ops.o ]; then
  ( g++ -O2 -std=c++17 -fPIC -ffp-contract=off -c host_ops.cpp -o ../_build/host_ops.o 2> ../_build/host_ops.log || { cat ../_build/host_ops.log; rm -f ../_build/host_ops.o; exit 1; } ) &
  pids="$pids $!"
fi
objs="$objs ../_build/host_ops.o"
# host-only C++: the text side of CT-Transformer punctuation (fa_punc_walk_host / fa_punc_infer's walk)
if [ ! -f ../_build/punc_text.o ] || [ punc_text.cpp -nt ../_build/punc_text.o ] || [ punc_text.h -nt ../_build/punc_text.o ]; then
  ( g++ -O2 -std=c++17 -fPIC -c punc_text.cpp -o ../_build/punc_text.o 2> ../_build/punc_text.log || { cat ../_build/punc_text.log; rm -f ../_build/punc_text.o; exit 1; } ) &
  pids="$pids $!"
fi
objs="$objs ../_build/punc_text.o"
for p in $pids; do wait $p || exit 1; done
$NVCC -gencode arch=compute_90a,code=sm_90a -shared -o ../libfunasr_b200.so $objs -lcudart
echo "built $(cd ..; pwd)/libfunasr_b200.so"
