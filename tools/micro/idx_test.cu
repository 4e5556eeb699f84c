#include <cstdio>
#include <cmath>
#include <cstdlib>
#include "../../jaero_b200/csrc/demod_device.cuh"
__global__ void k(const double *x, int *o, int n) { int i = blockIdx.x*blockDim.x+threadIdx.x; if (i<n) o[i] = jb::osc_index(x[i]); }
int main(){ const int n=1<<22; double *x; int *o; cudaMallocManaged(&x,n*8); cudaMallocManaged(&o,n*4);
 srand(3); for(int i=0;i<n;i++){ x[i]=rand()/(double)RAND_MAX*20010.0; if(i%7==0) x[i]=floor(x[i]); if(i%11==0) x[i]=nextafter(floor(x[i]),-1.0); if(i%13==0) x[i]=floor(x[i])+0.5; }
 x[0]=0; x[1]=19998.999999999996; x[2]=19999.0; x[3]=-0.0; x[4]=-1e-9; x[5]=20005.5; x[6]=0.49999999999999994; x[7]=1e300; x[8]=-5.0;
 k<<<(n+255)/256,256>>>(x,o,n); cudaDeviceSynchronize(); int bad=0;
 for(int i=0;i<n;i++){ if (!(x[i] > -2147483648.0 && x[i] < 2147483647.0)) continue;   /* out of int range: undefined on the host */ int t=(int)x[i]; if(t>=19999)t=0; if(t<0)t=19998; if(t!=o[i]){ if(bad<5)printf("mismatch x=%.17g ref %d got %d\n",x[i],t,o[i]); bad++; } }
 printf("osc_index mismatches: %d of %d\n", bad, n); return 0; }
