/* nrgbd_dev.h - development probes and A/B knobs of libnrgbd.so.
 *
 * NOT part of the product ABI (include/nrgbd.h): nothing here is bound by neuralrgbd_b200's product modules, the
 * knobs are process-global by design (they exist to compare kernel variants inside one process, tools/*.py) and
 * default to "off". No environment variable alters what a product entry point runs.
 */
#ifndef NRGBD_DEV_H_
#define NRGBD_DEV_H_
#include "nrgbd.h"
#ifdef __cplusplus
extern "C" {
#endif
void nrgbd_dev_set_bn_blocks_per_sm(int b);      /* BatchNorm pass: grid cap in blocks per SM (0 = chosen by tensor size: 8, or 32 from 64 MB) */
void nrgbd_dev_set_bn_unroll(int u);               /* BatchNorm pass: 16-byte vectors in flight per thread (1, 2 or 4; 0 = chosen by tensor size) */
void nrgbd_dev_conv_h2_set_flags(int flags);       /* tensor-core conv variants: flags listed next to g_h2_flags (conv_f16.cu) */
void nrgbd_dev_conv_h2_set_smem_cap_kb(int kb);    /* cap on the tensor-core conv's dynamic shared memory per CTA (0 = by plan) */
#ifdef __cplusplus
}
#endif
#endif /* NRGBD_DEV_H_ */
