// wgmma / TMA attention core (attn_tc.cu), dispatched from bb_flash_fwd / bb_flash_bwd (attn_flash.cu).
#pragma once
#include "../../include/bevbert_b200.h"

namespace bb {
namespace fat {
int tc_mode();
int set_tc_mode(int mode);
bool fwd_supported(const bb_flash_args* a);
int launch_fwd(const bb_flash_args* a, void* stream);
bool bwd_supported(const bb_flash_args* a);
int launch_bwd(const bb_flash_args* a, void* stream);
}  // namespace fat
}  // namespace bb
