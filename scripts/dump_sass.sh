#!/bin/bash
# Regenerates profiles/sass/*.sass from the built extension (cuobjdump -sass, one representative instantiation per kernel).
set -e
cd "$(dirname "$0")/.."
SO=$(ls torchft_b200/_K*.so | head -1)
OUT=profiles/sass
mkdir -p $OUT
dump() {  # name, regex on the mangled function name
  cuobjdump -sass -fun "$(cuobjdump -sass $SO | grep 'Function :' | sed 's/.*Function : //' | grep -E "$2" | head -1)" $SO > $OUT/$1.sass
  echo "$1: $(grep -cE '^\s+/\*[0-9a-f]{4}\*/' $OUT/$1.sass) instructions; $(grep -oE 'UBLKCP[.A-Z0-9]*|UTMALDG|UTMASTG|SYNCS[.A-Z0-9]*|LDGMC[.A-Z0-9_]*|STG\.E[.A-Z0-9]*\.SYS|MEMBAR[.A-Z.]*|REDG?[.A-Z0-9_]*' $OUT/$1.sass | sort | uniq -c | tr '\n' ' ')"
}
dump zero1_reduce_w8_p2p 'zero1_reduce_kernelILi8ELb0'
dump zero1_reduce_w8_nvls 'zero1_reduce_kernelILi8ELb1'
dump zero1_update_w8_p2p 'zero1_update_kernelILi8ELb0'
dump zero1_update_w8_nvls 'zero1_update_kernelILi8ELb1'
dump zero1_commit 'zero1_commit_kernel'
dump zero1_handshake 'zero1_handshake_kernel'
dump push_exchange 'push_exchange_kernel'
dump reduce_scatter_bf16_w8_sum 'reduce_scatter_kernelI13__nv_bfloat16Li8ELi0'
dump p2p_send 'p2p_send_kernel'
dump p2p_recv 'p2p_recv_kernel'
dump diloco_outer_bf16 'diloco_outer_kernelI13__nv_bfloat16'
dump heal_copy 'heal_copy_kernelE'
dump q8_allreduce_bf16_w8 'q8_allreduce_kernelI13__nv_bfloat16Li8'
dump allreduce_twoshot_bf16_w8_sum 'allreduce_twoshot_kernelI13__nv_bfloat16Li8ELi0'
dump allreduce_oneshot_bf16_w2_sum 'allreduce_oneshot_kernelI13__nv_bfloat16Li2ELi0'
dump allreduce_nvls_bf16 'allreduce_nvls_kernelI13__nv_bfloat16'
dump adamw 'adamw_kernel'
