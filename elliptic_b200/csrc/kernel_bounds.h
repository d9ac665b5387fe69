// kernel_bounds.h -- launch-bound choices shared by the translation units of libelliptic_b200.so
#pragma once

#ifndef EB_VERIFY_BLOCK
#define EB_VERIFY_BLOCK 128
#endif
#ifndef EB_VERIFY_MINBLOCKS
#define EB_VERIFY_MINBLOCKS 3
#endif
#ifndef EB_K256_VERIFY_MINBLOCKS
#define EB_K256_VERIFY_MINBLOCKS 4  // the secp256k1 verify kernel alone: 128 registers, four blocks per SM
#endif
#ifndef EB_SW_MINBLOCKS_BIG
#define EB_SW_MINBLOCKS_BIG 2     // 12- and 18-limb curves (p384, p521): 255 registers
#endif
#ifndef EB_SW_MINBLOCKS8
#define EB_SW_MINBLOCKS8 4        // 8-limb curves (p256, p224): four 128-thread blocks per SM (128 registers, a little
#endif                            // spill) measured faster than three blocks / 168 registers at N = 2^20
