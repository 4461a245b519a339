/* Drop-in for the reference's youtokentome/cpp/bpe.h (bpe.h:1-84): same namespace, types and signatures, bodies on the GPU. */
#pragma once
#include "../../../bpe_b200.h"
