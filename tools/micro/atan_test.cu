#include <cstdio>
#include <cmath>
#include <cstdlib>
#include "../../jaero_b200/csrc/demod_device.cuh"
__global__ void k(const double *y, const double *x, double *o, int n) { int i = blockIdx.x*blockDim.x+threadIdx.x; if (i<n) o[i] = jb::atan2_fast(y[i], x[i]); }
int main(){ const int n=1<<22; double *y,*x,*o; cudaMallocManaged(&y,n*8); cudaMallocManaged(&x,n*8); cudaMallocManaged(&o,n*8);
 srand(1); for(int i=0;i<n;i++){ double a=(rand()/(double)RAND_MAX*2-1), b=(rand()/(double)RAND_MAX*2-1); double s=pow(10.0,(rand()%40)-20); y[i]=a*s; x[i]=b*s*(i%3==0?1e-3:1); }
 y[0]=0;x[0]=1; y[1]=0;x[1]=-1; y[2]=-0.0;x[2]=-1; y[3]=1;x[3]=0; y[4]=0;x[4]=0; y[5]=1;x[5]=1; y[6]=-1;x[6]=1; y[7]=0.4375;x[7]=1; y[8]=0.6875;x[8]=1;
 k<<<(n+255)/256,256>>>(y,x,o,n); if (cudaDeviceSynchronize()!=cudaSuccess){printf("cuda error\n");return 1;}
 double maxulp=0; int bad=0; for(int i=0;i<n;i++){ double r=atan2(y[i],x[i]); double u=fabs(o[i]-r)/ (fabs(r)>0? (nextafter(fabs(r),1e300)-fabs(r)) : 4.9e-324); if(u>maxulp)maxulp=u; if (u>2.5) bad++; }
 printf("max ulp diff vs host atan2 %.2f, >2.5ulp: %d of %d; specials: %g %g %g %g %g\n", maxulp, bad, n, o[0],o[1],o[2],o[3],o[4]); return 0; }
